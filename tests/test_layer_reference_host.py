"""The per-kernel float64 references of oracle/layers.py and their bound, on the CPU.

* The wiring: the 26 references chained from the network input equal the oracle's U-Net (restate.unet_forward) run in
  float64, which pins the table's buffer ids, the concat order and the 1x1-before-upsample commutation.
* The bound accepts the kernels' arithmetic (split operands, three exact products, fp32 epilogue, split output).
* The bound rejects a kernel that loses a plane or a product (negative controls), for every kernel the fault applies
  to.  tests/test_gpu_layers.py applies the same bound to the engine's own buffers.
"""
import pytest
import torch

from oracle import layers, restate, synth

# Rejected fraction of the ReLU-active outputs per kernel and fault, measured on the `stored` chain (K = 3 random weights,
# seed 13, one phantom slice); the test asserts at least half of each.  Upsample and stem inputs are fp32, so their
# x_lo fault rounds the input to fp16.  The head's scores are checked against a bound propagated through the 1x1 and
# the log-softmax (oracle/layers.py: reference), which is looser, hence its lower fractions.
MEASURED = {
    "stem":                         {"x_lo": 0.968, "w_lo": 0.971, "out_lo": 0.937},
    "down_path.0.block.3":          {"x_lo": 0.890, "w_lo": 0.932, "lo_hi": 0.890, "out_lo": 0.710},
    "down_path.1.block.0":          {"x_lo": 0.942, "w_lo": 0.928, "lo_hi": 0.942, "out_lo": 0.755},
    "down_path.1.block.3":          {"x_lo": 0.838, "w_lo": 0.866, "lo_hi": 0.838, "out_lo": 0.653},
    "down_path.2.block.0":          {"x_lo": 0.923, "w_lo": 0.921, "lo_hi": 0.923, "out_lo": 0.706},
    "down_path.2.block.3":          {"x_lo": 0.750, "w_lo": 0.787, "lo_hi": 0.750, "out_lo": 0.571},
    "down_path.3.block.0":          {"x_lo": 0.893, "w_lo": 0.895, "lo_hi": 0.893, "out_lo": 0.648},
    "down_path.3.block.3":          {"x_lo": 0.640, "w_lo": 0.684, "lo_hi": 0.640, "out_lo": 0.448},
    "down_path.4.block.0":          {"x_lo": 0.853, "w_lo": 0.858, "lo_hi": 0.853, "out_lo": 0.588},
    "down_path.4.block.3":          {"x_lo": 0.803, "w_lo": 0.803, "lo_hi": 0.803, "out_lo": 0.510},
    "up_path.0.up.1":               {"x_lo": 0.931, "w_lo": 0.930, "lo_hi": 0.931},
    "upsample.0":                   {"x_lo": 0.995, "out_lo": 0.990},
    "up_path.0.conv_block.block.0": {"x_lo": 0.791, "w_lo": 0.792, "lo_hi": 0.791, "out_lo": 0.488},
    "up_path.0.conv_block.block.3": {"x_lo": 0.859, "w_lo": 0.861, "lo_hi": 0.859, "out_lo": 0.593},
    "up_path.1.up.1":               {"x_lo": 0.951, "w_lo": 0.952, "lo_hi": 0.951},
    "upsample.1":                   {"x_lo": 0.995, "out_lo": 0.991},
    "up_path.1.conv_block.block.0": {"x_lo": 0.853, "w_lo": 0.851, "lo_hi": 0.853, "out_lo": 0.590},
    "up_path.1.conv_block.block.3": {"x_lo": 0.898, "w_lo": 0.897, "lo_hi": 0.898, "out_lo": 0.670},
    "up_path.2.up.1":               {"x_lo": 0.965, "w_lo": 0.965, "lo_hi": 0.965},
    "upsample.2":                   {"x_lo": 0.995, "out_lo": 0.992},
    "up_path.2.conv_block.block.0": {"x_lo": 0.897, "w_lo": 0.896, "lo_hi": 0.897, "out_lo": 0.670},
    "up_path.2.conv_block.block.3": {"x_lo": 0.924, "w_lo": 0.926, "lo_hi": 0.924, "out_lo": 0.732},
    "up_path.3.up.1":               {"x_lo": 0.975, "w_lo": 0.975, "lo_hi": 0.975},
    "upsample.3":                   {"x_lo": 0.995, "out_lo": 0.993},
    "up_path.3.conv_block.block.0": {"x_lo": 0.926, "w_lo": 0.931, "lo_hi": 0.926, "out_lo": 0.734},
    "up_path.3.conv_block.block.3": {"x_lo": 0.122, "w_lo": 0.099, "lo_hi": 0.122},
}
# The emulation's worst ratio may reach about 1.75: the output split alone can be 2^-22 * |y| off, and |y| can equal M
# (the stem: 1.12 measured; the tensor-core layers stay below 0.41).  Half of tau leaves room for the truncating
# accumulation of the tensor core, which the emulation leaves out.
EMULATION_MAX = layers.TAU / 2


def threshold(kernel, fault):
    """The least rejected fraction the bound must show for `fault` in `kernel`: half the measured one."""
    return 0.5 * MEASURED[kernel][fault]


@pytest.fixture(scope="module")
def sd3():
    return synth.random_state_dict(3, seed=13, head_gain=0.3)


def _norm(S, seed):
    resized, _ = restate.preprocess(synth.phantom(S, seed=seed), resolution=[256, 256])
    return restate.normalise(resized)


@pytest.fixture(scope="module")
def stored(sd3):
    """The chain of one slice with every buffer held as the engine stores it: what each kernel reads."""
    return layers.chain(layers.network_input(_norm(1, 5)), sd3, as_stored=True)


def test_table_mirrors_the_engine():
    assert len(layers.KERNELS) == 26 and len(layers.ACT) == 29
    assert [k.mode for k in layers.KERNELS].count("Upsample") == 4
    assert sum(k.mode not in ("Upsample",) and k.name != "stem" for k in layers.KERNELS) == 21
    # every buffer is written by exactly one kernel, after it is read by none
    written = [d for k in layers.KERNELS for d in layers.outputs(k) if d != "scores"]
    assert sorted(written) == sorted(layers.ACT)
    seen = {"input"}
    for k in layers.KERNELS:
        assert k.src0 in seen and (k.src1 is None or k.src1 in seen), k.name
        seen.update(layers.outputs(k))
    assert set(MEASURED) == set(layers.BY_NAME)
    for name, m in MEASURED.items():
        assert set(m) == set(layers.faults_of(layers.BY_NAME[name])), name


def test_chain_equals_the_oracle_forward(sd3):
    """Two slices: the per-kernel references chained == restate.unet_forward on a float64 copy of the weights."""
    sd64 = {k: (v.to(torch.float64) if v.is_floating_point() else v) for k, v in sd3.items()}
    x = layers.network_input(_norm(2, 6))
    bufs = layers.chain(x, sd3)
    for name, (level, C, _) in layers.ACT.items():
        assert tuple(bufs[name].shape) == (2, C, 256 >> level, 256 >> level), name
    want = restate.unet_forward(x, sd64)
    err = float((bufs["scores"] - want).abs().max())
    print("chain vs unet_forward (float64): max |d score| = %.3e" % err)
    assert err <= 1e-12


@pytest.mark.parametrize("kernel", [k.name for k in layers.KERNELS])
def test_bound_accepts_the_emulated_kernel(sd3, stored, kernel):
    k = layers.BY_NAME[kernel]
    refs = layers.reference(k, stored, sd3)
    got = layers.emulate(k, stored, sd3)
    for out, r in refs.items():
        c = layers.check(got[out], r)
        print(layers.fmt(kernel, out, c))
        assert c.worst <= EMULATION_MAX, (kernel, out, c)


@pytest.mark.parametrize("kernel", [k.name for k in layers.KERNELS])
def test_bound_rejects_a_lost_plane(sd3, stored, kernel):
    k = layers.BY_NAME[kernel]
    refs = layers.reference(k, stored, sd3)
    for fault in layers.faults_of(k):
        got = layers.emulate(k, stored, sd3, fault)
        worst = min(layers.check(got[out], r, only_active=True).rejected for out, r in refs.items())
        print("%-30s %-6s rejected %.3f (threshold %.3f)" % (kernel, fault, worst, threshold(kernel, fault)))
        assert worst >= threshold(kernel, fault), (kernel, fault, worst)


def test_operand_split_is_the_engines():
    """split() restates split_f16: hi + lo * 2^-11 carries 22 bits, lo keeps its bits for small values."""
    t = torch.tensor([1.0, 1.0 + 2.0 ** -20, 3.0e-4, -65504.0, 0.1], dtype=torch.float64)
    hi, lo = layers.split(t)
    assert torch.all(hi == t.to(torch.float32).to(torch.float16).to(torch.float64))
    v = hi + lo
    assert float(((v - t.to(torch.float32).to(torch.float64)).abs() / t.abs()).max()) <= 2.0 ** -22
    with pytest.raises(ValueError):
        layers.split(torch.tensor([70000.0], dtype=torch.float64))
