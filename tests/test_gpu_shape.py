"""Mesh shape features on the GPU (LMInferer.shape, lm_shape_sums_dev, lm_max_diameters_dev) against the numpy statements
of lungmask_b200.shape: the cube counts, corner sums and moments must be equal, the squared diameters bit-identical to the
pruned restatement, and the features bit-identical to the host feature functions applied to the reference sums."""
import json
import math

import numpy as np
import pytest

from lungmask_b200 import shape as sh
from oracle import synth

pytestmark = pytest.mark.gpu

SPACING = (0.7, 0.8, 2.5)             # (x, y, z) mm; not dyadic
DYADIC = (0.703125, 0.703125, 1.25)   # every d^2 exact in float64


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


def _features_json(res):
    return json.dumps(res.to_dict())   # NaN-safe, bit-exact through repr


def check_exact(inf, mask, spacing=SPACING, rows=None):
    """The raw ABI results against the numpy statements, then LMInferer.shape against the host functions."""
    m8 = np.ascontiguousarray(mask).view(np.uint8) if mask.dtype == bool else mask
    tm = _cuda(m8)
    got = inf.engine.shape_sums_dev(tm.data_ptr(), m8.shape)
    counts, possum, moments = sh.cube_sums_host(m8)
    np.testing.assert_array_equal(got["cube_counts"], counts)
    np.testing.assert_array_equal(got["cube_possum"], possum)
    np.testing.assert_array_equal(got["moments"], moments)
    present = [int(x) for x in np.unique(m8) if x]
    for r in (present + [256]) if rows is None else rows:
        member = (m8 != 0) if r == 256 else (m8 == r)
        d2 = inf.engine.max_diameters_dev(tm.data_ptr(), m8.shape, r, spacing[::-1])
        np.testing.assert_array_equal(d2, sh.max_diameters_host(member, spacing), err_msg=str(r))
    res = inf.shape(mask, spacing=spacing)
    labels = sorted(set(present) | set(range(1, inf.engine.n_classes[0]))) + [256]
    assert [r.label for r in res.rows] == [("lung" if l == 256 else l) for l in labels]
    for row, l in zip(res.rows, labels):
        member = (m8 != 0) if l == 256 else (m8 == l)
        d2 = sh.max_diameters_host(member, spacing) if member.any() else np.zeros(4)
        want = sh.build_row(l, row.name, spacing, counts[l], possum[l], moments[l], d2)
        assert json.dumps(row.to_dict()) == json.dumps(want.to_dict()), l
    return res


def random_labels(seed, shape, labels):
    import scipy.ndimage as ndi
    rng = np.random.default_rng(seed)
    field = ndi.gaussian_filter(rng.standard_normal(shape), 1.5)
    m = (field > np.quantile(field, 0.4)).astype(np.uint8)
    region = ndi.gaussian_filter(rng.standard_normal(shape), 2.5)
    cuts = np.quantile(region, np.linspace(0, 1, labels + 1)[1:-1])
    return m * (np.searchsorted(cuts, region) + 1).astype(np.uint8)


@pytest.mark.parametrize("seed,shape,labels", [(0, (13, 27, 35), 1), (1, (20, 33, 47), 3), (2, (5, 64, 17), 6),
                                               (3, (31, 16, 32), 2), (4, (24, 40, 61), 5)])
def test_random_masks(inf, seed, shape, labels):
    check_exact(inf, random_labels(seed, shape, labels), SPACING if seed % 2 else DYADIC)


def test_touching_every_face_sheets_and_lines(inf):
    shape = (11, 19, 37)
    full = np.ones(shape, np.uint8)
    check_exact(inf, full)
    m = np.zeros(shape, np.uint8)
    m[:, 7, :] = 1          # a one-voxel sheet through the whole array
    m[4, :, 20] = 2         # a line along axis 1
    m[:, 15, 3] = 3         # a line along axis 0
    m[9, 2, 30] = 4         # a single voxel
    m[0, 0, :] = 5          # a line along x on the array's edge
    res = check_exact(inf, m)
    assert res[4]["Maximum3DDiameter"] == max(SPACING)
    rng = np.random.default_rng(5)
    check_exact(inf, rng.integers(0, 4, shape).astype(np.uint8))   # every label touches all six faces


def test_forty_labels(inf):
    """Labels beyond the rows privatised in shared memory go to global atomics."""
    rng = np.random.default_rng(6)
    m = np.zeros((18, 42, 50), np.uint8)
    for l in range(1, 41):
        z, y, x = rng.integers(0, 14), rng.integers(0, 36), rng.integers(0, 44)
        m[z:z + rng.integers(1, 5), y:y + rng.integers(1, 7), x:x + rng.integers(1, 7)] = l
    assert len(np.unique(m)) == 41
    check_exact(inf, m)


def test_empty_mask(inf):
    m = np.zeros((6, 17, 33), np.uint8)
    res = check_exact(inf, m)
    assert all(r.voxels == 0 and all(math.isnan(v) for v in r.features.values()) for r in res.rows)


def test_bool_mask(inf):
    m = random_labels(7, (12, 30, 45), 1) > 0
    a = check_exact(inf, m)
    b = inf.shape(m.astype(np.uint8), spacing=SPACING)
    assert _features_json(a) == _features_json(b)
    c = inf.shape(_cuda(m), spacing=SPACING)
    assert _features_json(a) == _features_json(c)


def test_input_paths(inf):
    import torch
    from lungmask_b200 import io as lio
    m = random_labels(8, (14, 38, 29), 3)
    a = inf.shape(m, spacing=SPACING)
    b = inf.shape(torch.from_numpy(m), spacing=SPACING)
    tm = _cuda(m)
    before = tm.clone()
    c = inf.shape(tm, spacing=SPACING)
    assert torch.equal(tm, before), "the CUDA mask was modified"
    d = inf.shape(m, image=lio.Volume(np.zeros(m.shape, np.int16), SPACING))
    assert _features_json(a) == _features_json(b) == _features_json(c) == _features_json(d)


def test_errors(inf):
    from lungmask_b200 import _native
    m = np.zeros((4, 5, 6), np.uint8)
    with pytest.raises(ValueError, match="spacing"):
        inf.shape(m)
    tm = _cuda(m)
    with pytest.raises(_native.NativeError, match="row"):
        inf.engine.max_diameters_dev(tm.data_ptr(), m.shape, 0, (1.0, 1.0, 1.0))
    with pytest.raises(_native.NativeError, match="spacing"):
        inf.engine.max_diameters_dev(tm.data_ptr(), m.shape, 1, (1.0, -1.0, 1.0))
    with pytest.raises(_native.NativeError, match="empty"):
        inf.engine.shape_sums_dev(tm.data_ptr(), (0, 5, 6))


def five_lobes(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    lobes = m.copy()
    lobes[(m == 1) & (z >= S // 2)] = 2
    lobes[(m == 1) & (z >= S // 2) & (y >= H // 2)] = 3
    lobes[(m == 2) & (z < S // 2)] = 4
    lobes[(m == 2) & (z >= S // 2)] = 5
    return m, lobes


def test_full_size(inf):
    """300x512x512: the two-lung phantom mask and a five-lobe split; sums exact, diameters equal to the CPU pruned
    restatement reduced to convex-hull vertices (dyadic spacing: every d^2 exact, so the reduction keeps the maximum)."""
    lungs, lobes = five_lobes(300, 512, 512)
    for m in (lungs, lobes):
        tm = _cuda(m)
        got = inf.engine.shape_sums_dev(tm.data_ptr(), m.shape)
        counts, possum, moments = sh.cube_sums_host(m)
        np.testing.assert_array_equal(got["cube_counts"], counts)
        np.testing.assert_array_equal(got["cube_possum"], possum)
        np.testing.assert_array_equal(got["moments"], moments)
        for r in [int(x) for x in np.unique(m) if x] + [256]:
            member = (m != 0) if r == 256 else (m == r)
            d2 = inf.engine.max_diameters_dev(tm.data_ptr(), m.shape, r, DYADIC[::-1])
            np.testing.assert_array_equal(d2, sh.max_diameters_host(member, DYADIC, hull=True), err_msg=str(r))


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
    out = str(tmp_path / ("shape." + ext))
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", wpath, "--noprogress", "--batchsize", "4", "--shape", out])
    inf = LMInferer(modelpath=wpath, tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.shape(inf.apply(v), image=v)
    assert want.spacing == (0.75, 0.5, 1.5)
    if ext == "json":
        assert json.load(open(out)) == json.loads(json.dumps(want.to_dict()))
    else:
        rows = list(csv.DictReader(open(out)))
        assert [r["label"] for r in rows] == [str(r.label) for r in want.rows]
        for r, w in zip(rows, want.rows):
            assert int(r["voxels"]) == w.voxels
            for k in sh.SHAPE_FEATURES:
                assert float(r[k]) == w.features[k] or math.isnan(w.features[k])
