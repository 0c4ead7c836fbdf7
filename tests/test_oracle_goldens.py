"""The CPU oracle (oracle/restate.py) against fixtures generated from the UNMODIFIED reference by
oracle/make_golden.py (tests/golden/).  Runs anywhere (no GPU, no reference checkout)."""
import json
import os
import zlib

import numpy as np
import torch

from oracle import make_golden, restate, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_preprocess_matches_reference_fixtures():
    cases = json.load(open(os.path.join(GOLD, "preprocess.json")))
    assert len(cases) == len(make_golden.PRE_CASES)
    for c in cases:
        vol = make_golden.pre_input(c["kind"], tuple(c["shape"]) if c["shape"] else None, c["seed"])
        out, boxes = restate.preprocess(vol, resolution=[256, 256])
        assert str(out.dtype) == c["dtype"]
        assert np.asarray(boxes).astype(int).tolist() == c["boxes"], c["kind"]
        assert [int(zlib.crc32(np.ascontiguousarray(s).tobytes())) for s in out] == c["crc32"], c["kind"]


def test_postprocess_matches_reference_fixtures():
    g = np.load(os.path.join(GOLD, "postprocess.npz"))
    for i, (S, K, seed, sp) in enumerate(make_golden.POST_CASES):
        lab = synth.label_noise_volume(S, K, seed=seed, speckle=sp)
        assert np.array_equal(lab, g[f"in{i}"]), "label generator drifted"
        assert np.array_equal(restate.postprocessing(lab), g[f"out{i}_plain"])
        assert np.array_equal(restate.postprocessing(lab, spare=[K - 1]), g[f"out{i}_spare"])
        assert np.array_equal(restate.postprocessing(lab, skip_below=1), g[f"out{i}_skip1"])


def test_forward_matches_reference_fixtures():
    g = np.load(os.path.join(GOLD, "forward.npz"))
    for K in (3, 6):
        sd = synth.random_state_dict(K, seed=10 + K)
        vol = synth.phantom(2, seed=21)
        tv, _ = restate.preprocess(vol, resolution=[256, 256])
        x = torch.as_tensor(restate.normalise(tv)[:, None], dtype=torch.float32)
        with torch.inference_mode():
            y = restate.unet_forward(x, sd).numpy()
        # weights come from numpy's PCG64 (machine independent); BN calibration and the forward are torch-CPU
        # fp32, so allow for a different SIMD width / thread count than the fixture's machine
        assert np.abs(y[:, :, 3::8, 5::8] - g[f"scores_K{K}"]).max() < 1e-4


def test_end_to_end_histograms():
    for c in json.load(open(os.path.join(GOLD, "e2e.json"))):
        sd = synth.random_state_dict(c["K"], seed=c["weights_seed"])
        vol = synth.phantom(*c["volume"], seed=c["volume_seed"])
        out = restate.inference(vol, sd, batch_size=2)
        hist = np.bincount(out.ravel(), minlength=c["K"])
        # random weights give speckled maps with argmax near-ties; a handful of voxels may flip across machines
        assert np.abs(hist - np.asarray(c["histogram"])).sum() <= 0.002 * out.size, (hist.tolist(), c["histogram"])
