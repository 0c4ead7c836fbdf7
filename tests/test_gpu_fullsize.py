"""BASELINE.json's full-size configurations through size-independent properties (the CPU oracle would need
minutes to hours at these sizes): slice independence of the per-slice stages, run-to-run determinism,
label range, and the fusion rule's invariants.  The exact full-size checks of C3 and C4 - every output voxel explained
by the network's labels through oracle.postfast - are in tests/test_gpu_post_fullsize.py."""
import os

import numpy as np
import pytest

from oracle import synth
from _parity import explain_fused, explain_inference, fmt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def big_engine():
    from lungmask_b200 import _native
    eng = _native.Engine(device=0, batch_capacity=33)
    yield eng
    eng.close()


def _load(eng, slot, K, seed):
    from lungmask_b200.mask import NativeModel
    m = NativeModel(synth.random_state_dict(K, seed=seed, head_gain=0.3))
    eng.load_weights(slot, m.blob, m.n_classes)


def _far_from_any_label(a, b):
    """Voxels whose whole 3x3 in-plane neighbourhood is background in both inputs and that lie outside the bounding
    box of every foreground voxel: hole filling and region merging cannot reach them."""
    fg = (a > 0) | (b > 0)
    far = np.ones(fg.shape, bool)
    if fg.any():
        idx = np.argwhere(fg)
        lo, hi = idx.min(0), idx.max(0) + 1
        far[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = False
    return far


def test_c3_ltrclobes_512_slices(big_engine):
    """C3: 6-class model, 512-slice 256x256 volume."""
    eng = big_engine
    _load(eng, 0, 6, seed=31)
    vol = synth.phantom(512, seed=40)
    raw = eng.apply_volume(0, vol, postprocess=False)
    assert raw.shape == vol.shape and raw.dtype == np.uint8 and raw.max() <= 5
    # per-slice stages are independent of how the volume is cut (mask.py:172-187 batches arbitrarily)
    halves = np.concatenate([eng.apply_volume(0, vol[:200], postprocess=False), eng.apply_volume(0, vol[200:], postprocess=False)])
    assert np.array_equal(raw, halves)
    assert np.array_equal(raw, eng.apply_volume(0, vol, postprocess=False))          # deterministic
    out = eng.apply_volume(0, vol)
    assert np.array_equal(out, eng.apply_volume(0, vol))
    assert set(np.unique(out)) <= set(range(6))
    # (a second application of the post-processing is NOT required to be the identity: a later label's filled holes
    #  can split an earlier label's component - parity with the oracle is checked at oracle-sized volumes instead)
    # every label kept by the post-processing already existed in the raw prediction
    assert set(np.unique(out)) <= set(np.unique(raw)) | {0}


def test_c4_fusion_300_slices(big_engine):
    """C4: LTRCLobes_R231 fusion on a 300-slice volume (two models, spare-label merge at original resolution)."""
    eng = big_engine
    _load(eng, 0, 6, seed=31)
    _load(eng, 1, 3, seed=32)
    vol = synth.phantom(300, seed=41)
    fused = eng.apply_fused(0, 1, vol)
    assert np.array_equal(fused, eng.apply_fused(0, 1, vol))
    # mask.py:341-342: the spare label (6) never survives.  (mask.py:230 zeroes the voxels the fill model calls
    # background BEFORE the post-processing, whose hole filling may legitimately paint some of them again.)
    assert fused.max() <= 5
    res_l = eng.apply_volume(0, vol)
    res_r = eng.apply_volume(1, vol)
    assert not np.any(fused[(res_l == 0) & (res_r == 0) & _far_from_any_label(res_l, res_r)])


def test_c2_r231_300_slices_through_lminferer(tmp_path):
    """C2 through the public surface: default LMInferer on a 300-slice volume == the capacity-33 engine."""
    import torch
    from lungmask_b200 import LMInferer
    sd = synth.random_state_dict(3, seed=33, head_gain=0.3)
    p = str(tmp_path / "r231_like.pth")
    torch.save(sd, p)
    inf = LMInferer(modelpath=p, tqdm_disable=True)
    vol = synth.phantom(300, seed=42)
    out = inf.apply(vol)
    assert out.shape == vol.shape and out.max() <= 2
    assert np.array_equal(out, inf.apply(vol))
    t = inf.engine.last_timings()
    assert t["kernel_launches"] > 9 * 26


# ---- the benchmarked configurations against the CPU oracle, with the bench's own weights ------------------------------
# (the oracle's fp32 forward runs at about 3 slices/s on the GPU box's host cores: C2 is compared in full, C3 / C4 on a
#  contiguous 64-slice sub-volume, sizes chosen with LM_FULLSIZE_SLICES / LM_SUBSAMPLE_SLICES)
def _bench_weights(K, seed):
    import bench
    return bench.get_weights(K, seed=seed)


def _load_sd(eng, slot, sd):
    from lungmask_b200.mask import NativeModel
    m = NativeModel(sd)
    eng.load_weights(slot, m.blob, m.n_classes)


def test_c2_bench_workload_against_oracle(big_engine):
    """C2 exactly as bench.py runs it (same phantom, same trained-looking weights), end to end against restate.inference:
    scores within 1e-4, every argmax flip on a sub-tolerance margin, integer stages bit-exact, every differing output
    voxel explained (tests/_parity.py)."""
    import bench
    S = int(os.environ.get("LM_FULLSIZE_SLICES", bench.S_VOL))
    sd = _bench_weights(3, 7)
    _load_sd(big_engine, 0, sd)
    vol = synth.phantom(bench.S_VOL, seed=100)[:S]
    rep = explain_inference(big_engine, 0, vol, sd, batch=20)
    print("C2 (%d slices, bench weights): %s" % (S, fmt(rep)))
    assert rep["dice"] >= 0.9999 or rep["label_flips"] > 0


def test_c3_c4_subvolume_against_oracle(big_engine):
    """C3 (6-class, batch 32) and C4 (fusion) with trained-looking weights on a contiguous sub-volume of the 512- /
    300-slice phantoms."""
    n = int(os.environ.get("LM_SUBSAMPLE_SLICES", "64"))
    sd6, sd3 = _bench_weights(6, 8), _bench_weights(3, 7)
    _load_sd(big_engine, 0, sd6)
    _load_sd(big_engine, 1, sd3)
    v3 = synth.phantom(512, seed=101)[256 - n // 2:256 + n // 2]
    rep = explain_inference(big_engine, 0, v3, sd6, batch=32)
    print("C3 (%d-slice sub-volume): %s" % (n, fmt(rep)))
    v4 = synth.phantom(300, seed=102)[150 - n // 2:150 + n // 2]
    rep = explain_fused(big_engine, 0, 1, v4, sd6, sd3, batch=20)
    print("C4 fusion (%d-slice sub-volume): %s" % (n, fmt(rep)))
    rep = explain_fused(big_engine, 0, 1, v4[:8], sd6, sd3, batch=20, postprocess=False)
    print("C4 fusion, volume_postprocessing=False (8 slices): %s" % fmt(rep))
