"""The engine's fp16 range scale groups (engine.cu: scale_group) as data, and the exact reparameterisation that moves one
group's activations by a power of two without changing the network.

Multiplying by 2^k the BatchNorm gamma / beta (or the 1x1 weight / bias) that produce a group's tensors and by 2^-k the
weights of every layer that reads them gives the same function in fp32, bit for bit: a power of two commutes with every
rounding (the BN fold included) as long as nothing is subnormal or overflows.  The group's tensors come out exactly 2^k
times larger, every other tensor and the scores are unchanged."""
from collections import OrderedDict

# group name (the engine's representative tensor) -> its split-plane tensors, the fp32 1x1 outputs that scale with them
# (read back by lm_debug_read_activation without a scale), the producers whose weight and bias go x 2^k and the weights
# of the consumers that go x 2^-k.
GROUPS = OrderedDict()
GROUPS["A0"] = dict(tensors=["A0"], fp32=[], up=["down_path.0.block.2"], down=["down_path.0.block.3.weight"])
for _i in range(4):
    GROUPS["S%d" % _i] = dict(
        tensors=["S%d" % _i, "P%d" % _i, "U%d" % (3 - _i)], fp32=["L%d" % (3 - _i)],
        up=["down_path.%d.block.5" % _i, "up_path.%d.up.1" % (3 - _i)],
        down=["down_path.%d.block.0.weight" % (_i + 1), "up_path.%d.conv_block.block.0.weight" % (3 - _i)])
    GROUPS["A%d" % (_i + 1)] = dict(tensors=["A%d" % (_i + 1)], fp32=[], up=["down_path.%d.block.2" % (_i + 1)],
                                    down=["down_path.%d.block.3.weight" % (_i + 1)])
GROUPS["B4"] = dict(tensors=["B4"], fp32=[], up=["down_path.4.block.5"], down=["up_path.0.up.1.weight"])
for _j in range(4):
    GROUPS["C%d" % _j] = dict(tensors=["C%d" % _j], fp32=[], up=["up_path.%d.conv_block.block.2" % _j],
                              down=["up_path.%d.conv_block.block.3.weight" % _j])
    if _j < 3:
        GROUPS["E%d" % _j] = dict(tensors=["E%d" % _j], fp32=[], up=["up_path.%d.conv_block.block.5" % _j],
                                  down=["up_path.%d.up.1.weight" % (_j + 1)])


def group_of(tensor):
    """The group a split-plane tensor belongs to."""
    for g, spec in GROUPS.items():
        if tensor in spec["tensors"]:
            return g
    raise KeyError(tensor)


def scaled_buffers(group):
    """Every buffer lm_debug_read_activation returns 2^k times larger for the group's variant."""
    return GROUPS[group]["tensors"] + GROUPS[group]["fp32"]


def rescale(sd, group, k):
    """-> a copy of state dict `sd` whose group `group` carries 2^k times its activations (k an integer); the same
    network in fp32 arithmetic."""
    spec = GROUPS[group]
    out = OrderedDict(sd)
    up, down = 2.0 ** k, 2.0 ** -k
    for p in spec["up"]:
        for s in (".weight", ".bias"):
            out[p + s] = sd[p + s] * up
    for key in spec["down"]:
        out[key] = sd[key] * down
    return out
