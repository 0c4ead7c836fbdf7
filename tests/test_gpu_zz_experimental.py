"""Alternative kernels of the forward against the default ones: each must reproduce the default path BIT FOR BIT (same
arithmetic in the same order, only the work assignment differs): stem_kernel vs stem_kernel_v2, upsample2x_kernel vs
upsample2x_cells_kernel, and the weight-multicast clusters (conv_tc.cu, MC = 2) vs one independent CTA per tile."""
import os

import numpy as np
import pytest

from oracle import restate, synth

pytestmark = pytest.mark.gpu


DEFAULTS = {"stem_v2": 3, "upsample_v2": 2, "weight_mcast": 0}


def _forward(engine, resized, **options):
    for k, v in options.items():
        engine.set_option(k, v)
    try:
        return engine.forward(3, resized, return_scores=True)
    finally:
        for k in options:
            engine.set_option(k, DEFAULTS[k])


@pytest.fixture(scope="module")
def setup(engine):
    from lungmask_b200.mask import NativeModel
    sd = synth.random_state_dict(3, seed=13, head_gain=0.3)
    m = NativeModel(sd)
    engine.load_weights(3, m.blob, m.n_classes)
    vol = synth.phantom(6, seed=21)      # 6 slices on a capacity-4 engine: a full wave and a 2-slice tail
    resized, _ = restate.preprocess(vol, resolution=[256, 256])
    return resized, _forward(engine, resized)


@pytest.mark.parametrize("option,value", [("stem_v2", 0), ("stem_v2", 1), ("stem_v2", 2), ("upsample_v2", 0), ("upsample_v2", 1), ("weight_mcast", 2)])
def test_experimental_kernel_is_bit_identical(engine, setup, option, value):
    """every alternative kernel against the default configuration"""
    resized, (labels, scores) = setup
    l2, s2 = _forward(engine, resized, **{option: value})
    assert np.array_equal(labels, l2)
    assert np.array_equal(scores, s2)
