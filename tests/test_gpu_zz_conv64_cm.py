"""The channel-major kernel of the 3x3 layers with 64 output channels (conv_tc.cu, conv_cm64_kernel, engine option
conv64_cm = 1, the default) against the BN = 64 kernel it replaces there (conv64_cm = 0): the same products summed in
the same order and the same epilogue operations, so labels and log-softmax scores must agree BIT FOR BIT - for both
class counts of the released models (the head's epilogue runs per class)."""
import numpy as np
import pytest

from oracle import restate, synth

pytestmark = pytest.mark.gpu


def _forward(engine, slot, resized, conv64_cm):
    engine.set_option("conv64_cm", conv64_cm)
    try:
        return engine.forward(slot, resized, return_scores=True)
    finally:
        engine.set_option("conv64_cm", 1)


@pytest.mark.parametrize("K", [3, 6])
def test_conv64_cm_is_bit_identical(engine, K):
    from lungmask_b200.mask import NativeModel
    slot = 2
    m = NativeModel(synth.random_state_dict(K, seed=20 + K, head_gain=0.3))
    engine.load_weights(slot, m.blob, m.n_classes)
    vol = synth.phantom(6, seed=22)      # 6 slices on a capacity-4 engine: a full wave and a 2-slice tail
    resized, _ = restate.preprocess(vol, resolution=[256, 256])
    l1, s1 = _forward(engine, slot, resized, 1)
    l0, s0 = _forward(engine, slot, resized, 0)
    assert s1.shape[1] == K
    assert np.array_equal(l1, l0)
    assert np.array_equal(s1, s0)
