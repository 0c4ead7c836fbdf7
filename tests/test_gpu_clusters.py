"""Low-attenuation cluster size distributions on the GPU (LMInferer.laa_clusters, lm_laa_clusters / lm_laa_clusters_dev)
against an oracle written here: scipy.ndimage.label (4 / 6 / 26 structure) plus np.bincount, per label and on the union.
Every row's (size, count) pairs, LAA voxel count and cluster count must be equal."""
import ctypes as C
import json

import numpy as np
import pytest
import scipy.ndimage as ndi

from oracle import synth

pytestmark = pytest.mark.gpu

CONNS = (4, 6, 26)


def structure(conn):
    if conn == 26:
        return np.ones((3, 3, 3), bool)
    if conn == 6:
        return ndi.generate_binary_structure(3, 1)
    s = np.zeros((3, 3, 3), bool)
    s[1] = ndi.generate_binary_structure(2, 1)
    return s


def oracle(vol, mask, t, conn):
    """{row: (laa_voxels, clusters, sizes, counts)} for every label value in the mask and "lung"."""
    v = np.asarray(vol).astype(np.float64)
    m = np.asarray(mask).astype(np.uint8)
    laa = (m > 0) & (v < t)
    out = {}
    for row in [int(x) for x in np.unique(m) if x] + ["lung"]:
        sel = laa if row == "lung" else laa & (m == row)
        lab, k = ndi.label(sel, structure(conn))
        sizes, counts = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
        out[row] = (int(sel.sum()), int(k), sizes.astype(np.int64), counts.astype(np.int64))
    return out


def check(res, want):
    for row, (vox, k, sizes, counts) in want.items():
        r = res[row]
        assert (r.laa_voxels, r.clusters) == (vox, k), (row, r.laa_voxels, r.clusters, vox, k)
        np.testing.assert_array_equal(r.sizes, sizes, err_msg=str(row))
        np.testing.assert_array_equal(r.counts, counts, err_msg=str(row))
        assert r.largest_voxels == (int(sizes[-1]) if sizes.size else 0)
    for r in res.rows:
        if r.label not in want:   # a model label absent from the mask
            assert r.laa_voxels == 0 and r.clusters == 0 and r.sizes.size == 0 and np.isnan(r.d)


@pytest.fixture(scope="module")
def inf():
    import tempfile
    import os
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=43, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _bytes(t):
    return t.cpu().numpy().tobytes()


def both_paths(inf, vol, mask, **kw):
    """laa_clusters() on numpy arrays and on CUDA tensors: bit-identical results; returns the numpy one."""
    a = inf.laa_clusters(vol, mask, **kw)
    tv, tm = _cuda(vol), _cuda(mask)
    bv, bm = tv.clone(), tm.clone()
    b = inf.laa_clusters(tv, tm, **kw)
    assert _bytes(tv) == _bytes(bv) and _bytes(tm) == _bytes(bm), "an input tensor was modified"
    assert json.dumps(a.to_dict()) == json.dumps(b.to_dict())
    return a


@pytest.fixture(scope="module")
def bullae():
    """40x160x192 int16: -850 +- 40 HU noise (LAA-950 speckle), labels 1 (x < 96) and 2 covering every voxel, spherical
    bullae of -990 HU: one straddling the label boundary, one centred on each face of the volume, a few inside."""
    S, H, W = 40, 160, 192
    rng = np.random.default_rng(61)
    vol = np.clip(-850 + 40 * rng.standard_normal((S, H, W)), -1024, 3071).astype(np.int16)
    mask = np.ones((S, H, W), np.uint8)
    mask[:, :, W // 2:] = 2
    z, y, x = np.ogrid[:S, :H, :W]
    centres = [(20, 80, W // 2, 9), (0, 60, 50, 6), (S - 1, 100, 140, 5), (25, 0, 40, 7), (12, H - 1, 150, 6),
               (30, 40, 0, 8), (8, 120, W - 1, 5), (15, 50, 60, 4), (30, 120, 130, 3)]
    for cz, cy, cx, r in centres:
        vol[(z - cz) ** 2 + (y - cy) ** 2 + (x - cx) ** 2 <= r * r] = -990
    return vol, mask


@pytest.mark.parametrize("conn", CONNS)
def test_bullae(inf, bullae, conn):
    vol, mask = bullae
    res = both_paths(inf, vol, mask, connectivity=conn)
    want = oracle(vol, mask, -950, conn)
    check(res, want)
    assert [r.label for r in res.rows] == [1, 2, "lung"] and res.connectivity == conn and res.threshold == -950
    # the straddling bulla is one cluster of the union and one in each label: the union's largest exceeds both labels'
    assert res["lung"].largest_voxels > max(res[1].largest_voxels, res[2].largest_voxels)
    assert res["lung"].clusters < res[1].clusters + res[2].clusters
    assert res["lung"].laa_voxels == res[1].laa_voxels + res[2].laa_voxels


def test_dense_overflow_seam(inf):
    """Clusters of exactly 4095, 4096 and 4097 voxels (the dense / overflow seam) and one of 1 024 000."""
    S, H, W = 24, 256, 256
    vol = np.full((S, H, W), -800, np.int16)
    vol[:16, :, :250] = -1000            # 16 x 256 x 250 = 1 024 000
    vol[18, :63, :65] = -1000            # 4095
    vol[20, 100:164, 100:164] = -1000    # 4096 + the voxel below: 4097
    vol[20, 100, 164] = -1000
    vol[22, 10:74, 10:74] = -1000        # 4096
    mask = np.ones((S, H, W), np.uint8)
    mask[22] = 2
    for conn in CONNS:
        res = both_paths(inf, vol, mask, connectivity=conn)
        check(res, oracle(vol, mask, -950, conn))
        sizes = set(res["lung"].sizes.tolist())
        assert {4095, 4096, 4097} <= sizes
        assert (1024000 in sizes) if conn != 4 else (64000 in sizes)


def test_speckle(inf):
    """White-noise LAA: more than 10^5 clusters of one voxel."""
    rng = np.random.default_rng(62)
    vol = np.where(rng.random((64, 256, 256)) < 0.035, -1000, -850).astype(np.int16)
    mask = np.ones(vol.shape, np.uint8)
    mask[:, :, 128:] = 2
    for conn in (6, 26):
        res = both_paths(inf, vol, mask, connectivity=conn)
        check(res, oracle(vol, mask, -950, conn))
    res = inf.laa_clusters(vol, mask, connectivity=6)
    assert res["lung"].sizes[0] == 1 and res["lung"].counts[0] > 100_000


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float_with_nans(inf, bullae, dtype):
    vol, mask = bullae
    rng = np.random.default_rng(63)
    v = (vol.astype(np.float64) + rng.uniform(-0.5, 0.5, vol.shape)).astype(dtype)
    v[rng.random(vol.shape) < 0.02] = np.nan
    v.flat[np.flatnonzero(mask == 1)[:4]] = (-950.0, np.nextafter(dtype(-950.0), dtype(-2000.0)), -5000.0, -np.inf)
    for conn in (6, 26):
        res = both_paths(inf, v, mask, connectivity=conn)
        check(res, oracle(v, mask, -950, conn))


def test_half_types(inf, bullae):
    """float16 / bfloat16 CUDA tensors are widened to float32: the clusters of the float32 tensor of those values."""
    import torch
    vol, mask = bullae
    rng = np.random.default_rng(64)
    v = torch.from_numpy(vol.astype(np.float32) + rng.uniform(-0.5, 0.5, vol.shape).astype(np.float32))
    tm = _cuda(mask)
    for dt in (torch.float16, torch.bfloat16):
        h = v.to(dt)
        got = inf.laa_clusters(h.to("cuda:0"), tm)
        check(got, oracle(h.float().numpy(), mask, -950, 6))
        assert json.dumps(inf.laa_clusters(h, mask).to_dict()) == json.dumps(got.to_dict())   # CPU tensor: numpy path


def test_integer_dtypes(inf, bullae):
    vol, mask = bullae
    wide = vol.astype(np.int64) * 3
    wide[mask == 2] -= 100000                     # beyond int16: all LAA
    wide.flat[np.flatnonzero(mask == 1)[::97]] = 2 ** 40           # not LAA at t = 3072; wrapped to int32: 0, LAA
    wide.flat[np.flatnonzero(mask == 1)[::89]] = -(2 ** 40)
    wide.flat[np.flatnonzero(mask == 1)[::83]] = 2 ** 32 + 4000    # wrapped to int32: 4000, still not LAA
    wide.flat[np.flatnonzero(mask == 2)[::79]] = 2 ** 32 + 3000    # not LAA; wrapped to int32: 3000, LAA
    # int32 at t = -1024: the values about -1275 are LAA only unclipped (the segmentation clips to [-1024, 600]).  A clip
    # to the int16 range cannot change `value < t` for t in [-1024, 3072]; wrap-around can, which the int64 case covers.
    i32 = (wide // 2).astype(np.int32)
    i32.flat[np.flatnonzero(mask == 2)[::71]] = 100000               # beyond int16, not LAA
    cases = [("bool", vol > -900, 1), ("uint8", (vol % 200).astype(np.uint8), 100),
             ("int8", (vol % 200 - 100).astype(np.int8), -30), ("int32", i32, -1024), ("int64", wide, 3072)]
    for name, v, t in cases:
        res = both_paths(inf, v, mask, threshold=t, connectivity=26)
        want = oracle(v, mask, t, 26)
        check(res, want)
        for row in (1, 2, "lung"):   # every case has LAA and non-LAA voxels in every row
            assert 0 < want[row][0] < int((mask > 0).sum() if row == "lung" else (mask == row).sum()), (name, row)


def test_forty_labels(inf, bullae):
    vol, _ = bullae
    rng = np.random.default_rng(65)
    mask = ((np.arange(vol.size) // 997) % 41).astype(np.uint8).reshape(vol.shape)
    mask[rng.random(vol.shape) < 0.3] = 0
    assert len(np.unique(mask)) == 41
    for conn in CONNS:
        res = both_paths(inf, vol, mask, connectivity=conn)
        check(res, oracle(vol, mask, -950, conn))
        assert [r.label for r in res.rows] == list(range(1, 41)) + ["lung"]


def test_empty_and_single_slice(inf, bullae):
    vol, mask = bullae
    none = inf.laa_clusters(np.zeros_like(vol), mask)       # nothing below -950
    assert [r.label for r in none.rows] == [1, 2, "lung"]
    for r in none.rows:
        assert r.laa_voxels == 0 and r.clusters == 0 and r.sizes.size == 0 and np.isnan(r.d) and r.largest_voxels == 0
    empty = inf.laa_clusters(vol, np.zeros_like(mask))     # no mask
    assert empty["lung"].laa_voxels == 0 and [r.label for r in empty.rows] == [1, 2, "lung"]
    for conn in CONNS:
        one = vol[19:20].copy()
        res = both_paths(inf, one, mask[19:20], connectivity=conn)
        check(res, oracle(one, mask[19:20], -950, conn))
        assert res["lung"].clusters > 0


def test_native_rows(inf, bullae):
    """The 257 rows of the C ABI: row 0 and absent labels zero, pairs ascending, row 256 the union; and the count of a
    row's LAA voxels equals lm_label_stats' below_count at the same threshold."""
    vol, mask = bullae
    m = mask.copy()
    m[:5] = 7
    eng = inf.engine
    for t in (-950, -900):
        res = eng.laa_clusters(vol, m, t, 6)
        assert res["laa_voxels"][0] == res["n_clusters"][0] == res["n_pairs"][0] == 0
        present = [1, 2, 7, 256]
        for r in range(257):
            if r not in present:
                assert res["laa_voxels"][r] == res["n_clusters"][r] == res["n_pairs"][r] == 0, r
        stats = eng.label_stats(vol, m, (), (t,))
        for r in present:
            s = res["sizes"][res["offsets"][r]:res["offsets"][r + 1]]
            c = res["counts"][res["offsets"][r]:res["offsets"][r + 1]]
            assert np.all(np.diff(s) > 0) and np.all(c > 0)
            assert int((s * c).sum()) == res["laa_voxels"][r] == stats["below_count"][r][0], (t, r)
            assert int(c.sum()) == res["n_clusters"][r]
        assert eng.last_timings()["kernel_launches"] > 0


def test_stream_ordering(inf, bullae):
    """The producer of the volume is still running when laa_clusters() is called: the engine waits on the caller's stream."""
    import torch
    vol, mask = bullae
    want = json.dumps(inf.laa_clusters(vol, mask).to_dict())
    src, tm = _cuda(vol), _cuda(mask)
    side = torch.cuda.Stream(device=0)
    for use_side in (True, False):
        t = torch.full(vol.shape, 0, dtype=torch.int16, device="cuda:0")
        torch.cuda.synchronize()
        with torch.cuda.stream(side if use_side else torch.cuda.default_stream(0)):
            torch.cuda._sleep(100_000_000)
            t.copy_(src)
            got = inf.laa_clusters(t, tm)
        assert json.dumps(got.to_dict()) == want, "side stream" if use_side else "default stream"
        torch.cuda.synchronize()


def test_volume_spacing_and_d(inf, bullae):
    from lungmask_b200 import io as lio
    from lungmask_b200.clusters import fit_d
    vol, mask = bullae
    spacing = (0.7, 0.8, 2.5)
    v = lio.Volume(vol, spacing, (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0))
    res = inf.laa_clusters(v, mask, min_cluster_voxels=2)
    assert res.spacing == spacing and res.min_cluster_voxels == 2
    ml = float(np.prod(spacing)) / 1000.0
    for r in res.rows:
        assert r.laa_volume_ml == r.laa_voxels * ml and r.largest_ml == r.largest_voxels * ml
        assert (r.d == fit_d(r.sizes, r.counts, 2)) or (np.isnan(r.d) and np.isnan(fit_d(r.sizes, r.counts, 2)))
    assert res["lung"].d > 0
    assert inf.laa_clusters(vol, mask)["lung"].laa_volume_ml is None


def test_errors(inf, bullae):
    import torch
    from lungmask_b200 import _native
    vol, mask = bullae
    tv, tm = _cuda(vol), _cuda(mask)
    with pytest.raises(ValueError):
        inf.laa_clusters(tv, mask)
    with pytest.raises(ValueError):
        inf.laa_clusters(vol, mask[:-1])
    with pytest.raises(ValueError):
        inf.laa_clusters(tv, tm[:-1])
    with pytest.raises(TypeError):
        inf.laa_clusters(vol, mask.astype(np.int16))
    with pytest.raises(ValueError):
        inf.laa_clusters(vol[0], mask[0])
    with pytest.raises(ValueError):
        inf.laa_clusters(vol, mask, threshold=-1025)
    with pytest.raises(ValueError):
        inf.laa_clusters(vol, mask, connectivity=18)
    with pytest.raises(TypeError):
        inf.laa_clusters(tv.to(torch.complex64), tm)
    eng = inf.engine
    with pytest.raises(_native.NativeError, match="threshold"):
        eng.laa_clusters(vol, mask, threshold=3073)
    with pytest.raises(_native.NativeError, match="connectivity"):
        eng.laa_clusters_dev(tv.data_ptr(), _native.DTYPE_I16, tm.data_ptr(), vol.shape, connectivity=8)
    with pytest.raises(_native.NativeError, match="not a CUDA pointer|not device memory"):
        eng.laa_clusters_dev(vol.ctypes.data, _native.DTYPE_I16, tm.data_ptr(), vol.shape)
    with pytest.raises(_native.NativeError, match="dtype"):
        eng.laa_clusters_dev(tv.data_ptr(), 99, tm.data_ptr(), vol.shape)
    with pytest.raises(_native.NativeError, match="empty volume"):
        eng.laa_clusters_dev(tv.data_ptr(), _native.DTYPE_I16, tm.data_ptr(), (0, 160, 192))
    with pytest.raises(_native.NativeError, match="2\\^32"):
        eng.laa_clusters_dev(tv.data_ptr(), _native.DTYPE_I16, tm.data_ptr(), (65536, 65536, 1))
    # a max_pairs below the bound is refused before any work: the outputs keep their sentinels
    L = _native.lib()
    cap = int(L.lm_laa_max_pairs(vol.size)) - 1
    outs = [np.full(257, -7, np.int64) for _ in range(3)] + [np.full(cap, -7, np.int64) for _ in range(2)]
    rc = L.lm_laa_clusters_dev(eng._h, C.c_void_p(tv.data_ptr()), _native.DTYPE_I16, C.c_void_p(tm.data_ptr()), *vol.shape, -950,
                               6, *[C.c_void_p(o.ctypes.data) for o in outs], cap, None)
    assert rc == -1 and "max_pairs" in L.lm_last_error().decode()
    assert all((o == -7).all() for o in outs)
    # the engine still works after the refusals
    check(inf.laa_clusters(tv, tm), oracle(vol, mask, -950, 6))


@pytest.mark.parametrize("ext", ["json", "csv"])
def test_cli(tmp_path, ext):
    import csv
    import torch
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main
    wpath = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=44, head_gain=0.3), wpath)
    vol = synth.phantom(6, 160, 176, seed=23)
    src = lio.Volume(vol, (0.75, 0.5, 1.5))
    inp = str(tmp_path / "in.mha")
    lio.save_mask(inp, vol, src)
    out = str(tmp_path / ("clusters." + ext))
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", wpath, "--noprogress", "--batchsize", "4", "--clusters", out,
          "--clusters-threshold", "-900", "--clusters-connectivity", "26"])
    inf = LMInferer(modelpath=wpath, tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.laa_clusters(v, inf.apply(v), threshold=-900, connectivity=26)
    if ext == "json":
        got = json.load(open(out))
        assert got == json.loads(json.dumps(want.to_dict()))
        assert got["threshold"] == -900 and got["connectivity"] == 26
    else:
        rows = list(csv.DictReader(open(out)))
        assert [r["label"] for r in rows] == [str(r.label) for r in want.rows]
        for r, w in zip(rows, want.rows):
            assert int(r["laa_voxels"]) == w.laa_voxels and int(r["clusters"]) == w.clusters
            assert float(r["laa_volume_ml"]) == w.laa_volume_ml
            assert float(r["d"]) == w.d or np.isnan(w.d)
