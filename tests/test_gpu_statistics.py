"""Per-label statistics on the GPU (LMInferer.statistics, lm_label_stats_dev) against a numpy oracle
written here: counts, min / max, fraction_below and numpy.percentile bit for bit, mean / std within 1e-12 relative."""
import json

import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu

Q = (0.0, 15.0, 50.0, 99.9, 100.0)
T = (-1024, -950, -910, 0, 3072)


def oracle(vol, mask, q=Q, t=T):
    """{row: dict} for every label value in the mask and "lung" (mask > 0), straight from numpy."""
    v64 = np.asarray(vol).astype(np.float64)
    mask = np.asarray(mask).astype(np.uint8)
    out = {}
    for row in [int(x) for x in np.unique(mask) if x] + ["lung"]:
        sel = mask > 0 if row == "lung" else mask == row
        vals = v64[sel]
        nan = np.isnan(vals)
        v = vals[~nan]
        r = {"voxels": int(sel.sum()), "nan_voxels": int(nan.sum())}
        if v.size:
            r.update(mean_hu=v.mean(), std_hu=v.std(), min_hu=v.min(), max_hu=v.max(),
                     percentile_hu={qq: np.percentile(v, qq) for qq in q}, fraction_below={tt: (v < tt).mean() for tt in t})
        out[row] = r
    return out


def _same_bits(a, b):
    return np.array(a, np.float64).view(np.int64) == np.array(b, np.float64).view(np.int64)


def check(stats, want):
    for row, w in want.items():
        g = stats[row]
        assert (g.voxels, g.nan_voxels) == (w["voxels"], w["nan_voxels"]), row
        if "mean_hu" not in w:
            assert np.isnan([g.mean_hu, g.std_hu, g.min_hu, g.max_hu]).all(), row
            assert all(np.isnan(x) for x in g.percentile_hu.values()) and all(np.isnan(x) for x in g.fraction_below.values())
            continue
        scale = max(abs(w["min_hu"]), abs(w["max_hu"]), 1.0)
        assert abs(g.mean_hu - w["mean_hu"]) <= 1e-12 * max(abs(w["mean_hu"]), scale * 1e-3), (row, g.mean_hu, w["mean_hu"])
        assert abs(g.std_hu - w["std_hu"]) <= 1e-12 * max(w["std_hu"], scale * 1e-3), (row, g.std_hu, w["std_hu"])
        assert _same_bits(g.min_hu, w["min_hu"]) and _same_bits(g.max_hu, w["max_hu"]), row
        for qq, x in w["percentile_hu"].items():
            assert _same_bits(g.percentile_hu[qq], x), (row, qq, g.percentile_hu[qq], x)
        for tt, x in w["fraction_below"].items():
            assert g.fraction_below[tt] == x, (row, tt)


@pytest.fixture(scope="module")
def weights(tmp_path_factory):
    import torch
    d = tmp_path_factory.mktemp("stats_weights")
    paths = {}
    for K in (3, 6):
        paths[K] = str(d / ("w%d.pth" % K))
        torch.save(synth.random_state_dict(K, seed=40 + K, head_gain=0.3), paths[K])
    return paths


@pytest.fixture(scope="module")
def inf6(weights):
    from lungmask_b200 import LMInferer
    return LMInferer(modelpath=weights[6], batch_size=4, tqdm_disable=True)


@pytest.fixture(scope="module")
def phantom():
    """40x200x216 int16 phantom with a 6-label blob mask: six ellipsoids, label 6 a single voxel."""
    vol = synth.phantom(40, 200, 216, seed=51)
    z, y, x = np.meshgrid(np.arange(40), np.arange(200), np.arange(216), indexing="ij")
    mask = np.zeros(vol.shape, np.uint8)
    centres = [(10, 60, 60), (10, 60, 150), (28, 140, 60), (28, 140, 150), (20, 100, 108)]
    for l, (cz, cy, cx) in enumerate(centres, 1):
        mask[((z - cz) / 9.0) ** 2 + ((y - cy) / 35.0) ** 2 + ((x - cx) / 30.0) ** 2 <= 1.0] = l
    mask[3, 5, 7] = 6
    return vol, mask


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def both_paths(inf, vol, mask, q=Q, t=T, **kw):
    """statistics() on numpy arrays and on CUDA tensors: checks that they agree field for field and returns the numpy one."""
    a = inf.statistics(vol, mask, percentiles=q, thresholds=t, **kw)
    tv, tm = _cuda(vol), _cuda(mask)
    bv, bm = tv.clone(), tm.clone()
    b = inf.statistics(tv, tm, percentiles=q, thresholds=t, **kw)
    assert _bytes(tv) == _bytes(bv) and _bytes(tm) == _bytes(bm), "an input tensor was modified"
    same(a, b, exact=np.issubdtype(np.asarray(vol).dtype, np.integer) or np.asarray(vol).dtype == bool)
    return a


def _bytes(t):
    return t.cpu().numpy().tobytes()   # NaN-safe equality


def same(a, b, exact):
    """Two results agree: every field equal; mean / std of float volumes (float64 sums in no fixed order) within 1e-12."""
    da, db = a.to_dict(), b.to_dict()
    if not exact:
        for ra, rb in zip(da["rows"], db["rows"]):
            for k in ("mean_hu", "std_hu"):
                if ra[k] is not None and rb[k] is not None and abs(ra[k] - rb[k]) <= 1e-12 * max(abs(ra[k]), 1.0):
                    rb[k] = ra[k]
    assert json.dumps(da) == json.dumps(db)


def test_int16_six_labels(inf6, phantom):
    vol, mask = phantom
    s = both_paths(inf6, vol, mask)
    check(s, oracle(vol, mask))
    assert [r.label for r in s.rows] == [1, 2, 3, 4, 5, 6, "lung"]
    assert s[6].voxels == 1 and s[6].percentile_hu[15.0] == float(vol[3, 5, 7])
    # integer volumes: exact sums, so a second call gives identical results
    assert json.dumps(inf6.statistics(vol, mask, percentiles=Q, thresholds=T).to_dict()) == json.dumps(s.to_dict())


def test_values_outside_the_bins(inf6, phantom):
    """int16 extremes and values beyond [-1024, 3071] put order statistics into the under- and overflow bins."""
    vol, mask = phantom
    v = vol.copy()
    rng = np.random.default_rng(5)
    for l in (1, 2, 3):
        idx = np.flatnonzero(mask == l)
        pick = rng.choice(idx, size=idx.size // 3, replace=False)
        v.flat[pick[: len(pick) // 2]] = rng.integers(-32768, -1025, len(pick) // 2)
        v.flat[pick[len(pick) // 2:]] = rng.integers(3072, 32768, len(pick) - len(pick) // 2)
    v.flat[np.flatnonzero(mask == 1)[:2]] = (-32768, 32767)
    s = both_paths(inf6, v, mask)
    check(s, oracle(v, mask))
    assert s[1].min_hu == -32768 and s[1].max_hu == 32767


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float_with_nans(inf6, phantom, dtype):
    vol, mask = phantom
    rng = np.random.default_rng(7)
    v = (vol.astype(np.float64) + rng.uniform(-0.5, 0.5, vol.shape)).astype(dtype)
    v[mask == 2] *= np.float64(1.37)
    nan_at = rng.random(vol.shape) < 0.01
    v[nan_at] = np.nan
    v.flat[np.flatnonzero(mask == 3)[:5]] = (-5000.25, 4000.5, -1024.0, -0.0, 3071.75)
    s = both_paths(inf6, v, mask)
    check(s, oracle(v, mask))
    assert s[1].nan_voxels == int((nan_at & (mask == 1)).sum()) > 0


def test_half_types(inf6, phantom):
    """float16 / bfloat16 CUDA tensors are widened to float32: the same statistics as the float32 tensor of those values."""
    import torch
    vol, mask = phantom
    rng = np.random.default_rng(8)
    v = torch.from_numpy((vol.astype(np.float32) + rng.uniform(-0.5, 0.5, vol.shape).astype(np.float32)))
    tm = _cuda(mask)
    for dt in (torch.float16, torch.bfloat16):
        h = v.to(dt)
        got = inf6.statistics(h.to("cuda:0"), tm, percentiles=Q, thresholds=T)
        check(got, oracle(h.float().numpy(), mask))
        cpu = inf6.statistics(h, mask, percentiles=Q, thresholds=T)      # CPU tensor: the numpy path
        same(cpu, got, exact=False)


def test_integer_dtypes(inf6, phantom):
    import torch
    vol, mask = phantom
    wide = vol.astype(np.int64) * 3
    wide[mask == 4] += 100000
    wide.flat[np.flatnonzero(mask == 5)[:2]] = (-(2 ** 40), 2 ** 40)
    cases = {"bool": vol > -500, "uint8": (vol % 200).astype(np.uint8), "int8": (vol % 100).astype(np.int8),
             "int32": wide.astype(np.int32) // 2, "int64": wide}
    for name, v in cases.items():
        check(both_paths(inf6, v, mask), oracle(v, mask))
    assert inf6.statistics(_cuda(cases["int32"]), _cuda(mask))[4].max_hu > 50000
    # a bool mask is the label-1 mask
    s = inf6.statistics(_cuda(vol), _cuda(mask > 0), percentiles=Q, thresholds=T)
    check(s, oracle(vol, (mask > 0).astype(np.uint8)))
    assert s[1].voxels == int((mask > 0).sum()) and torch.equal(_cuda(mask > 0), _cuda(mask) > 0)


def test_forty_labels(inf6, phantom):
    """More labels than fit shared memory: the global-memory histograms and selection state."""
    vol, _ = phantom
    rng = np.random.default_rng(9)
    mask = ((np.arange(vol.size) // 997) % 41).astype(np.uint8).reshape(vol.shape)
    mask[rng.random(vol.shape) < 0.3] = 0
    assert len(np.unique(mask)) == 41
    check(both_paths(inf6, vol, mask), oracle(vol, mask))
    vf = (vol + rng.uniform(-0.5, 0.5, vol.shape)).astype(np.float32)
    check(both_paths(inf6, vf, mask), oracle(vf, mask))


def test_empty_model_labels_and_union(inf6, phantom):
    vol, mask = phantom
    m = np.where(mask <= 2, mask, 0).astype(np.uint8)
    s = inf6.statistics(vol, m)
    assert [r.label for r in s.rows] == [1, 2, 3, 4, 5, "lung"]   # the 6-class model's labels 1..5 are always reported
    for l in (3, 4, 5):
        assert s[l].voxels == 0 and np.isnan(s[l].mean_hu) and np.isnan(s[l].percentile_hu[15.0])
        assert np.isnan(s[l].fraction_below[-950])
    assert s["lung"].voxels == s[1].voxels + s[2].voxels
    check(s, oracle(vol, m, (15.0,), (-950,)))
    empty = inf6.statistics(vol, np.zeros_like(m))
    assert empty["lung"].voxels == 0 and np.isnan(empty["lung"].mean_hu)


def test_stream_ordering(inf6, phantom):
    """The producer of the volume is still running when statistics() is called: the engine waits on the caller's stream."""
    import torch
    vol, mask = phantom
    want = json.dumps(inf6.statistics(vol, mask).to_dict())
    src, tm = _cuda(vol), _cuda(mask)
    side = torch.cuda.Stream(device=0)
    for use_side in (True, False):
        t = torch.full(vol.shape, -1000, dtype=torch.int16, device="cuda:0")
        torch.cuda.synchronize()
        with torch.cuda.stream(side if use_side else torch.cuda.default_stream(0)):
            torch.cuda._sleep(100_000_000)
            t.copy_(src)
            got = inf6.statistics(t, tm)
        assert json.dumps(got.to_dict()) == want, "side stream" if use_side else "default stream"
        torch.cuda.synchronize()


def test_volume_end_to_end(inf6, phantom):
    """apply(Volume) of a RAS-oriented volume with non-unit spacing, then statistics(Volume, mask)."""
    from lungmask_b200 import io as lio
    vol, _ = phantom
    ras = (-1.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 1.0)
    spacing = (0.7, 0.8, 2.5)
    v = lio.Volume(np.ascontiguousarray(vol[:, ::-1, ::-1]), spacing, (0.0, 0.0, 0.0), ras)
    mask = inf6.apply(v)
    assert mask.max() > 0
    s = inf6.statistics(v, mask)
    assert s.spacing == spacing
    for r in s.rows:
        assert r.volume_ml == r.voxels * float(np.prod(spacing)) / 1000.0
    check(s, oracle(v.array, mask, (15.0,), (-950,)))
    assert inf6.statistics(v, mask, spacing=(1.0, 1.0, 1.0))["lung"].volume_ml == s["lung"].voxels / 1000.0
    assert inf6.statistics(vol, mask)["lung"].volume_ml is None


def test_errors_dev(inf6, phantom):
    import torch
    from lungmask_b200 import _native
    vol, mask = phantom
    tv, tm = _cuda(vol), _cuda(mask)
    with pytest.raises(ValueError):
        inf6.statistics(tv, mask)                       # mixed placements
    with pytest.raises(ValueError):
        inf6.statistics(vol, tm)
    with pytest.raises(ValueError):
        inf6.statistics(tv, tm.cpu())
    with pytest.raises(ValueError):
        inf6.statistics(vol, mask[:-1])                 # shapes
    with pytest.raises(ValueError):
        inf6.statistics(tv, tm[:-1])
    with pytest.raises(TypeError):
        inf6.statistics(vol, mask.astype(np.int16))     # mask dtype
    with pytest.raises(TypeError):
        inf6.statistics(tv, tm.to(torch.int32))
    with pytest.raises(ValueError):
        inf6.statistics(vol[0], mask[0])                # not 3-D
    with pytest.raises(ValueError):
        inf6.statistics(tv[0], tm[0])
    with pytest.raises(ValueError):
        inf6.statistics(vol, mask, percentiles=(101.0,))
    with pytest.raises(ValueError):
        inf6.statistics(vol, mask, thresholds=(-1025,))
    with pytest.raises(TypeError):
        inf6.statistics(vol, mask, thresholds=(-950.5,))
    with pytest.raises(ValueError):
        inf6.statistics(vol, mask, spacing=(1.0, 1.0))
    with pytest.raises(TypeError):
        inf6.statistics(tv.to(torch.complex64), tm)
    # the C entry points refuse bad arguments before any kernel runs
    eng = inf6.engine
    with pytest.raises(_native.NativeError, match="not in \\[0,100\\]"):
        eng.label_stats_dev(tv.data_ptr(), _native.DTYPE_I16, tm.data_ptr(), vol.shape, percentiles=(-1.0,))
    with pytest.raises(_native.NativeError, match="threshold"):
        eng.label_stats_dev(tv.data_ptr(), _native.DTYPE_I16, tm.data_ptr(), vol.shape, thresholds=(3073,))
    with pytest.raises(_native.NativeError, match="not a CUDA pointer|not device memory"):
        eng.label_stats_dev(vol.ctypes.data, _native.DTYPE_I16, tm.data_ptr(), vol.shape)
    with pytest.raises(_native.NativeError, match="not a CUDA pointer|not device memory"):
        eng.label_stats_dev(tv.data_ptr(), _native.DTYPE_I16, mask.ctypes.data, vol.shape)
    with pytest.raises(_native.NativeError, match="dtype"):
        eng.label_stats_dev(tv.data_ptr(), 99, tm.data_ptr(), vol.shape)
    with pytest.raises(_native.NativeError, match="empty volume"):
        eng.label_stats_dev(tv.data_ptr(), _native.DTYPE_I16, tm.data_ptr(), (0, 200, 216))
    # the engine still works after the refusals
    check(inf6.statistics(tv, tm), oracle(vol, mask, (15.0,), (-950,)))


@pytest.mark.parametrize("ext", ["json", "csv"])
def test_cli(tmp_path, weights, ext):
    import csv
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main
    vol = synth.phantom(6, 160, 176, seed=22)
    src = lio.Volume(vol, (0.75, 0.5, 1.5))
    inp = str(tmp_path / "in.mha")
    lio.save_mask(inp, vol, src)
    out = str(tmp_path / ("stats." + ext))
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", weights[3], "--noprogress", "--batchsize", "4", "--statistics", out])
    inf = LMInferer(modelpath=weights[3], tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.statistics(v, inf.apply(v))
    assert want["lung"].voxels > 0
    if ext == "json":
        got = json.load(open(out))
        assert got == json.loads(json.dumps(want.to_dict()))
        assert got["percentiles"] == [15.0] and got["thresholds"] == [-950]
    else:
        rows = list(csv.DictReader(open(out)))
        assert [r["label"] for r in rows] == [str(r.label) for r in want.rows]
        for r, w in zip(rows, want.rows):
            assert int(r["voxels"]) == w.voxels and float(r["volume_ml"]) == w.volume_ml
            assert float(r["percentile_15"]) == w.percentile_hu[15.0] or np.isnan(w.percentile_hu[15.0])
            assert float(r["fraction_below_-950"]) == w.fraction_below[-950] or np.isnan(w.fraction_below[-950])
            assert float(r["mean_hu"]) == w.mean_hu or np.isnan(w.mean_hu)
    # --nopostprocess
    out2 = str(tmp_path / ("stats_np." + ext))
    main([inp, str(tmp_path / "mask2.nii.gz"), "--modelpath", weights[3], "--noprogress", "--nopostprocess", "--statistics", out2])
    inf.volume_postprocessing = False
    want2 = inf.statistics(v, inf.apply(v))
    if ext == "json":
        assert json.load(open(out2)) == json.loads(json.dumps(want2.to_dict()))
