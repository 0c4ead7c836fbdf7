"""Validates the oracle against the reference ITSELF: tests/golden/reference.json holds what the unmodified reference
(run with the stand-ins of oracle/standins.py) returned on the seeded inputs below - its state_dict schema and digests
(dtype, shape, CRC32) of its outputs, written by `python -m oracle.make_golden --reference`."""
import json
import os

import numpy as np
import pytest

from oracle import make_golden, restate, synth

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference.json")))


def test_reference_known_answer_tests_through_standins():
    """tests/test_utils.py:58-63,73-107,124-159 of the reference: its verbatim assertions, on the restatement."""
    m = np.zeros((10, 10, 10), dtype=np.uint8)
    m[2:8, 3:7, 4:6] = 1
    assert tuple(restate.bbox_3D(m, margin=2)) == (0, 10, 1, 9, 2, 8)
    img = np.full((10, 10), dtype=np.int16, fill_value=-1000)
    img[2:8, 3:7] = 1
    img[9, 9] = 1
    li = np.zeros((1, 6, 6), dtype=np.uint8)
    li[0] = np.asarray([[0, 0, 0, 0, 0, 0], [0, 1, 1, 2, 2, 0], [0, 2, 0, 3, 1, 0], [0, 4, 4, 4, 0, 0], [0, 4, 0, 4, 0, 0], [0, 4, 4, 4, 0, 0]])
    gt = [[0, 0, 0, 0, 0, 0], [0, 1, 1, 2, 2, 0], [0, 1, 0, 3, 2, 0], [0, 4, 4, 4, 0, 0], [0, 4, 0, 4, 0, 0], [0, 4, 4, 4, 0, 0]]
    vol = np.tile(li, (2, 1, 1))
    assert np.sum(restate.simple_bodymask(img)) == 24
    c2, b2 = restate.crop_and_resize(img, width=20, height=20)
    assert tuple(b2) == (2, 3, 8, 7) and c2.shape == (20, 20) and np.sum(c2) == 400
    out = restate.reshape_mask(np.full((10, 10), dtype=np.uint8, fill_value=1), (2, 2, 22, 22), origsize=(30, 30))
    assert out.shape == (30, 30) and np.sum(out) == 400
    assert np.all(restate.postprocessing(vol, spare=[], skip_below=1)[0] == gt)
    assert restate.postprocessing(vol, spare=[3], skip_below=1)[0][2, 3] == 2
    assert restate.postprocessing(vol, spare=[3], skip_below=3)[0][2, 1] == 0


def test_state_dict_schema_is_the_reference_layout():
    for K in (3, 6):
        sch = synth.schema(K)
        assert [[k, list(s)] for k, s, _ in sch] == GOLD["schema"][str(K)]
        assert len(sch) == 227


@pytest.mark.parametrize("shape,seed", make_golden.REF_PRE_CASES)
def test_preprocess_equals_reference(shape, seed):
    want = GOLD["preprocess"][make_golden.REF_PRE_CASES.index((shape, seed))]
    r, br = restate.preprocess(synth.phantom(*shape, seed=seed), resolution=[256, 256])
    assert [make_golden.digest(r), make_golden.digest(np.asarray(br))] == want


@pytest.mark.parametrize("S,K,seed", make_golden.REF_POST_CASES)
def test_postprocessing_equals_reference(S, K, seed):
    want = GOLD["post"][make_golden.REF_POST_CASES.index((S, K, seed))]
    lab = synth.label_noise_volume(S, K, seed=seed, speckle=2e-3)
    assert make_golden.digest(restate.postprocessing(lab)) == want[0]
    assert make_golden.digest(restate.postprocessing(lab, spare=[K - 1])) == want[1]


def test_forward_and_apply_equal_reference():
    sd, vol = make_golden.forward_case()
    taps = {}
    assert make_golden.digest(restate.inference(vol, sd, batch_size=2, taps=taps)) == GOLD["forward"]["apply"]
    assert make_golden.digest(np.asarray(taps["scores"], dtype=np.float32)) == GOLD["forward"]["scores"]


def test_preprocess_equals_reference_on_ragged_and_noisy_volumes():
    """slices smaller than the 128 x 128 thumbnail, non-square and odd sizes, volumes without a clear body"""
    vols = make_golden.ragged_volumes()
    assert len(vols) == len(GOLD["ragged"])
    for vol, want in zip(vols, GOLD["ragged"]):
        r, br = restate.preprocess(vol, resolution=[256, 256])
        assert [make_golden.digest(r), make_golden.digest(np.asarray(br))] == want, vol.shape


def test_postprocessing_equals_reference_sweep():
    """random sizes, class counts and speckle levels x the spare / skip_below combinations of utils.py:272"""
    cases = list(make_golden.post_sweep_cases())
    assert len(cases) == len(GOLD["post_sweep"])
    for (seed, K, lab), want in zip(cases, GOLD["post_sweep"]):
        for (spare, skip), w in zip(make_golden.REF_POST_SPARE_SKIP, want):
            spare = [K - 1 if c == -1 else c for c in spare]
            got = restate.postprocessing(lab.copy(), spare=list(spare), skip_below=skip)
            assert make_golden.digest(got) == w, (seed, K, spare, skip)
