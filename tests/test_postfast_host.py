"""oracle.postfast against oracle.restate: the fast restatement of utils.postprocessing must give the same output, bit
for bit, and the same taps (regions0, regions1, mapped), so that the GPU post-processing can be compared with it at
sizes restate cannot reach.  Also: its emulation of the merge loop's batch schedule against tests/test_merge_batches.py,
and what the speed-up is."""
import time

import numpy as np
import pytest

from oracle import postfast, restate, synth
from test_merge_batches import batched


def _same(lab, spare=(), skip_below=3):
    ta, tb = {}, {}
    want = restate.postprocessing(lab, spare=spare, skip_below=skip_below, taps=ta)
    got = postfast.postprocessing(lab, spare=spare, skip_below=skip_below, taps=tb)
    for k in ("regions0", "regions1", "mapped"):
        assert np.array_equal(ta[k], tb[k]), (k, lab.shape, spare, skip_below, int((ta[k] != tb[k]).sum()))
    assert np.array_equal(want, got), (lab.shape, spare, skip_below, int((want != got).sum()))
    return tb


def _variants(lab, K):
    for spare in ([], [K - 1], [1, 2]):
        for skip in (3, 1, 2):
            _same(lab, spare, skip)


# ---- the label volumes tests/test_gpu_stages.py post-processes ------------------------------------------------------
# (skip_below = 1 makes every speckle a candidate; restate then relabels the whole volume thousands of times, so that
#  variant stops at volumes of about half a million voxels to keep this file near a minute)
@pytest.mark.parametrize("S,K,speckle", [(12, 3, 2e-3), (9, 6, 2e-3), (1, 3, 2e-3), (2, 6, 1e-3), (5, 3, 0.0), (40, 6, 5e-4)])
def test_gpu_stage_noise_volumes(S, K, speckle):
    lab = synth.label_noise_volume(S, K, seed=S + K, speckle=speckle)
    for kw in ({}, {"spare": [K - 1]}, {"spare": [1, 2]}) + (({"skip_below": 1},) if S < 40 else ()):
        _same(lab, **kw)


def test_gpu_stage_other_volumes():
    _same(np.zeros((3, 32, 48), np.uint8))
    _same(np.ones((2, 16, 16), np.uint8))        # no background: np.unique(mapped)[1:] skips label 1
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 4, size=(4, 24, 24)).astype(np.uint8)
    _same(noise)
    _same(noise, spare=[3])
    _same(rng.integers(0, 3, size=(1, 40, 40)).astype(np.uint8))
    lab = synth.label_noise_volume(6, 6, seed=2, speckle=1e-3, H=200, W=312)
    _same(lab)
    _same(lab, spare=[6])
    rng = np.random.default_rng(7)
    for lab in (synth.label_noise_volume(12, 3, seed=5, speckle=0.0), synth.label_noise_volume(12, 6, seed=15, speckle=2e-3),
                synth.label_noise_volume(7, 3, seed=25, speckle=2e-2, H=130, W=97),
                rng.integers(0, 4, size=(5, 33, 47)).astype(np.uint8)):
        _same(lab)
    noise = np.random.default_rng(9).integers(0, 4, size=(4, 40, 40)).astype(np.uint8)
    _same(noise)
    _same(noise, spare=[3])
    _same(np.random.default_rng(13).integers(0, 3, size=(2, 30, 30)).astype(np.uint8))


def test_gpu_stage_merge_volumes():
    rng = np.random.default_rng(21)
    for lab in (synth.label_noise_volume(16, 3, seed=31, speckle=2e-2),
                synth.label_noise_volume(10, 6, seed=32, speckle=5e-3, H=200, W=312),
                rng.integers(0, 4, size=(6, 48, 48)).astype(np.uint8)):
        for kw in ({}, {"spare": [int(lab.max())]}) + (({"skip_below": 1},) if lab.size < 600_000 else ()):
            _same(lab, **kw)


# ---- seeded random small volumes ------------------------------------------------------------------------------------
def test_random_small_volumes():
    rng = np.random.default_rng(11)
    for trial in range(216):
        shape = (int(rng.integers(1, 5)), int(rng.integers(3, 14)), int(rng.integers(3, 14)))
        K = int(rng.integers(2, 6))
        if trial % 3 == 0:
            lab = rng.integers(0, K, size=shape)
        elif trial % 3 == 1:
            lab = np.where(rng.random(shape) < 0.7, 1, rng.integers(0, K, size=shape))
        else:
            lab = (rng.random(shape) < 0.5).astype(int) * rng.integers(1, K, size=shape)
        _variants(lab.astype(np.uint8), K)


# ---- hand-built edge cases ------------------------------------------------------------------------------------------
def _tie_volume():
    """Region C (label 3, 3 voxels, not the label's record) between B (label 1) above and D (label 2) below."""
    lab = np.zeros((3, 12, 12), np.uint8)
    lab[:, 9:12, 9:12] = 3          # the label-3 record holder: id 1 (its first voxel is the first in raster order)
    lab[1, 3, 3:6] = 1              # B: id 2
    lab[1, 4, 3:6] = 3              # C: id 3
    lab[1, 5, 3:6] = 2              # D: id 4
    return lab


def test_equal_ring_counts_lowest_id_wins():
    lab = _tie_volume()
    t = _same(lab)
    assert t["regions0"][1, 4, 3] == 3 and t["regions1"][1, 4, 3] == 2      # B and D both touch 3 voxels: B (id 2)
    _variants(lab, 4)


def test_best_neighbour_id_equal_to_a_spare_value_is_skipped():
    lab = _tie_volume()
    lab[1, 5, 5] = 0                # D now touches 2 voxels, B still 3
    t = _same(lab, spare=[2])       # region id 2 (B) equals the spare label value 2: C goes to D (id 4)
    assert t["regions1"][1, 4, 3] == 4
    assert t["mapped"][1, 4, 3] == 0                                        # D is label 2, the spare label
    t = _same(lab)
    assert t["regions1"][1, 4, 3] == 2


def test_equal_area_regions_lowest_id_sets_the_record():
    lab = np.zeros((4, 10, 10), np.uint8)
    lab[0:2, 1:3, 1:3] = 1
    lab[2:4, 6:8, 6:8] = 1
    t = _same(lab)
    assert t["mapped"][0, 1, 1] == 1 and t["mapped"][3, 7, 7] == 0          # to_label only for the first of equal areas
    _variants(lab, 2)


def test_merges_lifting_the_target_to_the_record_and_chains():
    lab = np.zeros((3, 20, 20), np.uint8)
    lab[:, 0:4, 0:5] = 1            # label-1 record holder, 60 voxels
    lab[:, 8:11, 0:4] = 1           # T: 36 voxels
    lab[:, 11:13, 0:4] = 2          # A: 24 voxels of label 2, touches only T -> T reaches the record (60): no candidate
    lab[:, 15:20, 15:20] = 2        # the label-2 record holder
    lab[1, 8:11, 8] = 3             # a: touches b only
    lab[1, 8:11, 9:11] = 4          # b: touches a and c; 6 + 3 voxels, still below its label's record
    lab[:, 8:11, 11:16] = 1         # c: a label-1 region
    lab[0, 0:4, 19] = 3             # the label-3 record
    lab[2, 16:19, 0:4] = 4          # the label-4 record
    for skip in (1, 2, 3):
        _same(lab, skip_below=skip)
        _same(lab, spare=[3], skip_below=skip)
    t = _same(lab)
    T, c = t["regions0"][1, 9, 1], t["regions0"][1, 9, 12]
    assert t["regions1"][1, 11, 1] == T and t["regions1"][1, 9, 1] == T   # A merged into T, T stayed
    assert t["regions1"][1, 9, 8] == c and t["regions1"][1, 9, 9] == c    # a -> b -> c


def test_candidate_without_non_zero_neighbour_keeps_its_id():
    lab = np.zeros((5, 12, 12), np.uint8)
    lab[:, 0:4, 0:4] = 1
    lab[2, 8, 7:11] = 1             # isolated, not the record
    t = _same(lab)
    assert t["regions1"][2, 8, 7] == t["regions0"][2, 8, 7]
    _variants(lab, 2)


def test_regions_touching_all_faces():
    lab = np.ones((4, 6, 7), np.uint8)
    lab[1:3, 2:4, 2:5] = 2
    lab[0, 0, 0] = lab[3, 5, 6] = lab[0, 5, 0] = lab[3, 0, 6] = 2
    lab[2, 0, 3] = lab[1, 5, 3] = lab[2, 3, 0] = lab[1, 2, 6] = 3
    lab[0, 2:5, 2:4] = 3
    lab[3, 1:3, 1:3] = 3
    _variants(lab, 4)


def test_holes_open_to_the_first_or_last_slice_are_not_filled():
    lab = np.zeros((5, 10, 10), np.uint8)
    lab[:, 2:8, 2:8] = 1
    lab[0:2, 4:6, 4:6] = 0          # open at slice 0
    lab[4, 3:5, 3:5] = 0            # open at the last slice
    lab[2, 6, 6] = 0                # enclosed
    out = restate.postprocessing(lab)
    assert out[0, 4, 4] == 0 and out[1, 4, 4] == 0 and out[4, 3, 3] == 0 and out[2, 6, 6] == 1
    _variants(lab, 2)


def test_single_slice_area_closing_63_and_64_pixels():
    lab = np.zeros((1, 40, 40), np.uint8)
    lab[0, 2:38, 2:38] = 1
    lab[0, 5:12, 5:14] = 0          # 63 px: closed
    lab[0, 20:28, 20:28] = 0        # 64 px: kept
    out = restate.postprocessing(lab)
    assert out[0, 6, 6] == 1 and out[0, 22, 22] == 0
    _variants(lab, 2)


def test_two_largest_components_tie():
    lab = np.zeros((3, 16, 16), np.uint8)
    lab[1, 1:3, 1:5] = 1            # P: 8 voxels
    lab[1, 6, 6:11] = 1             # Q: 5 voxels ...
    lab[1, 7, 6:9] = 2              # ... + a 3-voxel label-2 candidate that touches only Q: 8 voxels of label 1
    lab[:, 12:15, 12:15] = 2
    out = _same(lab) and restate.postprocessing(lab)
    assert out[1, 1, 1] == 0 and out[1, 6, 6] == 1 and out[1, 7, 6] == 1   # argsort(...)[-1]: the later component
    _variants(lab, 3)


# ---- the batch schedule diagnostics ---------------------------------------------------------------------------------
def test_schedule_matches_merge_batch_emulation(monkeypatch):
    """postfast's record of the multi-CTA schedule equals tests/test_merge_batches.py's emulation of it (no window
    limit there: volumes of fewer than MC_WINDOW regions)."""
    monkeypatch.setattr(postfast, "MC_SMALL", 0)
    rng = np.random.default_rng(3)
    seen = 0
    for trial in range(30):
        shape = (int(rng.integers(2, 5)), int(rng.integers(6, 16)), int(rng.integers(6, 16)))
        K = int(rng.integers(2, 5))
        lab = np.where(rng.random(shape) < 0.7, 1, rng.integers(0, K, size=shape)).astype(np.uint8)
        for B in (4, 256):
            monkeypatch.setattr(postfast, "MC_BMAX", B)
            for spare, skip in (([], 3), ([K - 1], 1), ([1, 2], 2)):
                want = []
                batched(lab, spare, skip, B=B, stats=want)
                d = {}
                postfast.postprocessing(lab, spare=spare, skip_below=skip, diag=d)
                assert d["batches"] == want, (trial, B, spare, skip)
                seen += sum(want)
    assert seen > 1000


def test_diagnostics_count_neighbour_ids():
    lab = np.zeros((3, 60, 90), np.uint8)
    lab[1, :, :60] = 1
    lab[1, 2:58:2, 2:58:2] = 2      # 784 single label-2 voxels (below skip_below) inside a label-1 sheet
    lab[:, :, 70:90] = 1            # a larger label-1 region: the sheet is a candidate
    d = {}
    postfast.postprocessing(lab, diag=d)
    assert d["max_ids"] == 784 and d["regions"] > postfast.MC_SMALL and d["schedule"] == "batched"
    _same(lab)


# ---- speed ----------------------------------------------------------------------------------------------------------
def test_speedup_on_a_speckled_volume():
    """skip_below = 1: every speckle is a merge candidate, and restate relabels the whole volume for each one."""
    lab = synth.label_noise_volume(24, 3, seed=3, speckle=2e-2, H=128, W=128)
    t0 = time.perf_counter()
    want = restate.postprocessing(lab, skip_below=1)
    t1 = time.perf_counter()
    d = {}
    got = postfast.postprocessing(lab, skip_below=1, diag=d)
    t2 = time.perf_counter()
    assert np.array_equal(want, got)
    print("24x128x128, %d regions, %d candidates: restate %.2f s, postfast %.2f s (%.0fx)"
          % (d["regions"], d["candidates"], t1 - t0, t2 - t1, (t1 - t0) / (t2 - t1)))
    assert t2 - t1 < (t1 - t0) / 5
