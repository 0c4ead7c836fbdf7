"""The GPU post-processing at benchmark sizes against oracle.postfast, bit for bit, stage by stage.

restate.postprocessing costs O(candidates x voxels), so tests/test_gpu_stages.py can only compare small volumes with it.
oracle.postfast gives the same result (tests/test_postfast_host.py) fast enough for 300- and 512-slice volumes and for
the fusion's 300 x 512 x 512 post-processing.  Every case compares the engine's parity taps (lm_set_option
"post_debug_stage": 2 = region ids & 255, 3 = merged region ids & 255, 1 = the label map before step 6), then the output,
and names the first stage that differs.  Each case asserts from postfast's diagnostics that it reaches the gate of the
merge loop it is there for (postproc.cu: MC_SMALL, MC_WINDOW, MC_BMAX, MC_HASH, the region sort's shared-memory limit,
the region-table overflow).  LM_POST_FULLSIZE_SLICES=n caps every volume at n slices for a quick run (the gate
assertions that need the full size are then skipped)."""
import os
import time

import numpy as np
import pytest

from oracle import postfast, restate, synth

pytestmark = pytest.mark.gpu

_CAP = int(os.environ.get("LM_POST_FULLSIZE_SLICES", "0"))
_FULL = _CAP <= 0
_DEFAULTS = {"merge_ctas": 0, "ccl_rule": 1, "post_region_capacity": 1 << 16}
_STAGES = ((2, "region ids & 255"), (3, "merged region ids & 255"), (1, "label map before step 6"), (0, "output"))
_ROWS = []


def _slices(S):
    return min(S, _CAP) if _CAP > 0 else S


@pytest.fixture(scope="module", autouse=True)
def _table():
    yield
    print("\n%-34s %-26s %8s %8s %7s %6s %7s %7s %7s" % ("case", "options", "regions", "cands", "max_ids", "batch", "batches",
                                                          "cpu_s", "gpu_s"))
    for r in _ROWS:
        print("%-34s %-26s %8d %8d %7d %6d %7d %7.1f %7.2f" % r)


@pytest.fixture(scope="module")
def model_engine():
    from lungmask_b200 import _native
    eng = _native.Engine(device=0, batch_capacity=33)
    yield eng
    eng.close()


def _reference(lab, spare=(), skip_below=3):
    taps, diag = {}, {}
    t0 = time.perf_counter()
    out = postfast.postprocessing(lab, spare=spare, skip_below=skip_below, taps=taps, diag=diag)
    diag["cpu_s"] = time.perf_counter() - t0
    want = {2: (taps["regions0"] & 255).astype(np.uint8), 3: (taps["regions1"] & 255).astype(np.uint8), 1: taps["mapped"], 0: out}
    return want, diag


def _check(engine, name, lab, want, diag, spare=(), skip_below=3, options=None):
    """engine.postprocess(lab) through every tap, then the output, with `options` set for the call."""
    options = dict(options or {})
    gpu = 0.0
    try:
        for k, v in options.items():
            engine.set_option(k, v)
        for stage, what in _STAGES:
            engine.set_option("post_debug_stage", stage)
            t0 = time.perf_counter()
            got = engine.postprocess(lab, spare=spare, skip_below=skip_below)
            gpu = time.perf_counter() - t0
            bad = int(np.count_nonzero(got != want[stage]))
            assert bad == 0, "%s %s: the %s differs in %d of %d voxels" % (name, options, what, bad, lab.size)
    finally:
        engine.set_option("post_debug_stage", 0)
        for k in options:
            engine.set_option(k, _DEFAULTS[k])
    b = diag["batches"]
    _ROWS.append((name, ",".join("%s=%s" % kv for kv in options.items()) or "-", diag["regions"], diag["candidates"],
                  diag["max_ids"], max(b) if b else 0, len(b), diag["cpu_s"], gpu))


# ---- label_noise_volume at 300 and 512 slices -----------------------------------------------------------------------
@pytest.mark.parametrize("S,K,speckle,kw,options", [
    (300, 3, 2e-2, {}, ({}, {"merge_ctas": 1}, {"merge_ctas": 5}, {"ccl_rule": 0}, {"post_region_capacity": 4096})),
    (300, 3, 2e-2, {"skip_below": 1}, ({}, {"merge_ctas": 5})),
    (300, 6, 0.0, {}, ({}, {"ccl_rule": 0})),
    (512, 6, 2e-3, {"spare": [5]}, ({}, {"merge_ctas": 1})),
    (512, 3, 2e-2, {}, ({}, {"post_region_capacity": 100000})),
])
def test_label_noise_volume(engine, S, K, speckle, kw, options):
    S = _slices(S)
    lab = synth.label_noise_volume(S, K, seed=S + K, speckle=speckle)
    want, diag = _reference(lab, **kw)
    name = "noise S=%d K=%d speckle=%g %s" % (S, K, speckle, "".join("%s=%s" % i for i in kw.items()))
    for opt in options:
        _check(engine, name, lab, want, diag, options=opt, **kw)
    if _FULL and speckle > 0:
        assert diag["sort"] == "global" and diag["schedule"] == "batched" and diag["regions"] > 10 * postfast.MC_WINDOW
        assert len(diag["batches"]) > 10
    if _FULL and speckle >= 2e-2:
        assert diag["regions"] > 65536 and postfast.MC_BMAX in diag["batches"]
        for opt in options:
            if "post_region_capacity" in opt:
                assert diag["regions"] > opt["post_region_capacity"]    # the tables overflow and the call runs again


# ---- one non-record region with more than MC_HASH distinct neighbours -----------------------------------------------
def test_neighbour_table_overflow(engine):
    """A label-1 sheet (not the label's largest region) sown with 3,844 single voxels of labels 2-5: below skip_below,
    they stay distinct regions, so the sheet's ring holds 3,844 ids and the batch member that decides it hands over to
    the serial routine."""
    rng = np.random.default_rng(4)
    lab = np.zeros((5, 128, 256), np.uint8)
    lab[2, :, :128] = 1
    lab[2, 2:126:2, 2:126:2] = rng.integers(2, 6, size=(62, 62))
    lab[:, :, 160:256] = 1                   # the label-1 record holder
    lab[0:2, 10:20, 10:20] = 2                # records for labels 2-5, so that their larger blobs are candidates too
    lab[0:2, 30:40, 10:20] = 3
    lab[0:2, 50:60, 10:20] = 4
    lab[0:2, 70:80, 10:20] = 5
    lab[3:5, 2:126:8, 2:126:8] = 3            # more regions before the sheet in the order
    for kw in ({}, {"spare": [5]}):
        want, diag = _reference(lab, **kw)
        assert diag["max_ids"] > postfast.MC_HASH and diag["serial"] >= 1 and diag["schedule"] == "batched"
        for opt in ({}, {"merge_ctas": 5}, {"merge_ctas": 1}):
            _check(engine, "neighbour ids > MC_HASH %s" % kw, lab, want, diag, options=opt, **kw)


# ---- the sequential loop up to MC_SMALL regions, the batched kernel above ---------------------------------------------
def _blobs(n):
    """Two lungs (labels 1, 2) and n 3-voxel label-2 blobs inside lung 1, pairwise separated: 2 + n regions."""
    lab = np.zeros((4, 64, 64), np.uint8)
    lab[:, 4:60, 4:30] = 1
    lab[:, 4:60, 34:60] = 2
    spots = [(z, y, x) for z in (0, 2) for y in range(6, 59, 2) for x in range(6, 27, 4)]
    for z, y, x in spots[:n]:
        lab[z, y, x:x + 3] = 2
    return lab


@pytest.mark.parametrize("regions", [postfast.MC_SMALL - 1, postfast.MC_SMALL, postfast.MC_SMALL + 1, postfast.MC_SMALL + 40])
def test_small_region_counts(engine, regions):
    lab = _blobs(regions - 2)
    for kw in ({}, {"spare": [2]}, {"skip_below": 4}):
        want, diag = _reference(lab, **kw)
        assert diag["regions"] == regions
        assert diag["schedule"] == ("sequential" if regions <= postfast.MC_SMALL else "batched")
        for opt in ({}, {"merge_ctas": 1}, {"merge_ctas": 5}):
            _check(engine, "%d regions %s" % (regions, kw), lab, want, diag, options=opt, **kw)


# ---- whole volumes: network labels -> post-processing -> original resolution, and the fusion --------------------------
def _load(eng, slot, sd):
    from lungmask_b200.mask import NativeModel
    m = NativeModel(sd)
    eng.load_weights(slot, m.blob, m.n_classes)


def _explain_inference(eng, engine, slot, vol, name):
    """apply_volume == reshape_mask(postfast(the engine's network labels)), with the post-processing compared stage by
    stage in between -> the result at the input's resolution."""
    resized, boxes = eng.preprocess(vol)
    labels = eng.forward(slot, resized)
    want, diag = _reference(labels)
    _check(engine, name, labels, want, diag)
    expect = np.stack([restate.reshape_mask(want[0][i], boxes[i], vol.shape[1:]) for i in range(vol.shape[0])]).astype(np.uint8)
    got = eng.apply_volume(slot, vol)
    bad = int(np.count_nonzero(got != expect))
    assert bad == 0, "%s: apply_volume differs from the explained composition in %d voxels" % (name, bad)
    return got


def _explain_fusion(eng, engine, res_l, res_r, vol, name):
    pre, spare = eng.fuse(res_l, res_r)
    want_pre, want_spare = restate.fuse_pre(res_l, res_r)
    assert spare == int(want_spare) and np.array_equal(pre, want_pre), name
    want, diag = _reference(want_pre, spare=[spare])
    _check(engine, name, want_pre, want, diag, spare=[spare])
    got = eng.apply_fused(0, 1, vol)
    bad = int(np.count_nonzero(got != want[0]))
    assert bad == 0, "%s: apply_fused differs from fuse + postprocess in %d voxels" % (name, bad)


def test_fusion_at_original_resolution(model_engine, engine):
    """A 300 x 512 x 512 phantom through a 6-class and a 3-class model: the fusion's post-processing runs on 78 M
    voxels at the input's resolution."""
    _load(model_engine, 0, synth.random_state_dict(6, seed=31, head_gain=0.3))
    _load(model_engine, 1, synth.random_state_dict(3, seed=32, head_gain=0.3))
    vol = synth.phantom(_slices(300), 512, 512, seed=43)
    res_l = model_engine.apply_volume(0, vol)
    res_r = model_engine.apply_volume(1, vol)
    _explain_fusion(model_engine, engine, res_l, res_r, vol, "fusion %dx512x512" % vol.shape[0])


def _bench_weights(K, seed):
    import bench
    return bench.get_weights(K, seed=seed)


def test_c3_explained_at_full_size(model_engine, engine):
    """C3 (6-class model, 512 slices, bench weights): every output voxel explained by the network's labels."""
    _load(model_engine, 0, _bench_weights(6, 8))
    vol = synth.phantom(_slices(512), seed=101)
    _explain_inference(model_engine, engine, 0, vol, "C3 %d slices" % vol.shape[0])


def test_c4_explained_at_full_size(model_engine, engine):
    """C4 (fusion of a 6- and a 3-class model, 300 slices, bench weights): both inferences and the fusion explained."""
    _load(model_engine, 0, _bench_weights(6, 8))
    _load(model_engine, 1, _bench_weights(3, 7))
    vol = synth.phantom(_slices(300), seed=102)
    res_l = _explain_inference(model_engine, engine, 0, vol, "C4 base %d slices" % vol.shape[0])
    res_r = _explain_inference(model_engine, engine, 1, vol, "C4 fill %d slices" % vol.shape[0])
    _explain_fusion(model_engine, engine, res_l, res_r, vol, "C4 fusion %d slices" % vol.shape[0])
