"""The premise of tests/test_gpu_zz_range_groups.py, checked on the CPU: the groups of tests/_range_groups.py are the
engine's fp16 range scale groups, and moving one group by 2^k (tests/_range_groups.rescale) leaves the network unchanged
in fp32, bit for bit, while the group's tensors in the float64 chain come out exactly 2^k times larger."""
import os
import re

import numpy as np
import pytest
import torch

from _range_groups import GROUPS, group_of, rescale, scaled_buffers
from oracle import layers, restate, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = (8, 24, 40)


def _split_tensors():
    return [name for name, (_, _, split) in layers.ACT.items() if split]


def _engine_scale_group():
    """engine.cu scale_group(): {member: representative} of its switch (every other tensor is its own group)."""
    src = open(os.path.join(ROOT, "lungmask_b200", "csrc", "engine.cu")).read()
    body = re.search(r"int scale_group\(int a\) \{(.*?)\n\}", src, re.S).group(1)
    out = {}
    for cases, rep in re.findall(r"((?:case \w+: )+)return (\w+);", body):
        for m in re.findall(r"case (\w+):", cases):
            out[m.rstrip("_")] = rep.rstrip("_")
    assert out, "scale_group's switch was not found"
    return out


def test_groups_partition_the_split_tensors():
    members = [t for spec in GROUPS.values() for t in spec["tensors"]]
    assert len(GROUPS) == 17
    assert sorted(members) == sorted(_split_tensors()), "every split tensor in exactly one group"
    assert len(set(members)) == len(members)
    for g, spec in GROUPS.items():
        assert g in spec["tensors"]
        for t in spec["fp32"]:
            assert not layers.ACT[t][2]


def test_groups_match_the_engine_and_the_network():
    rep = _engine_scale_group()
    for t in _split_tensors():
        assert group_of(t) == rep.get(t, t), t
    # the rule behind the groups: a block output and its pooled copy leave one epilogue, and the two halves of a
    # virtual concat feed one accumulator with one in_unscale; nothing else needs to share a scale
    parent = {t: t for t in _split_tensors()}

    def find(t):
        while parent[t] != t:
            t = parent[t]
        return t
    for k in layers.KERNELS:
        for a, b in ((k.dst, k.dst_pool), (k.src0, k.src1)):
            if a in parent and b in parent:
                parent[find(a)] = find(b)
    for t in _split_tensors():
        assert all((find(t) == find(u)) == (group_of(t) == group_of(u)) for u in _split_tensors()), t
    # the fp32 1x1 output that an upsampled member is made from scales with the group
    for g, spec in GROUPS.items():
        made_from = {k.src0 for k in layers.KERNELS if k.mode == "Upsample" and k.dst in spec["tensors"]}
        assert made_from == set(spec["fp32"]), g


def test_rescale_touches_only_the_named_parameters():
    sd = synth.random_state_dict(3, seed=7, calibrate_on=np.zeros((1, 256, 256), np.float32) + 0.5)
    for g, spec in GROUPS.items():
        v = rescale(sd, g, 8)
        changed = {key for key in sd if not torch.equal(sd[key], v[key])}
        want = {p + s for p in spec["up"] for s in (".weight", ".bias")} | set(spec["down"])
        assert want <= set(sd) and changed == want, g


@pytest.fixture(scope="module")
def net():
    sd = synth.random_state_dict(3, seed=23, head_gain=0.3)
    resized, _ = restate.preprocess(synth.phantom(2, seed=29), resolution=[256, 256])
    norm = restate.normalise(resized)
    _, scores = restate.forward_volume(norm, sd, batch_size=2, return_scores=True)
    ch = layers.chain(layers.network_input(norm[:1]), sd)   # float64: one slice (about 3 s each on 8 CPU cores)
    return sd, norm, scores, ch


@pytest.mark.parametrize("group", list(GROUPS))
def test_rescaled_group_is_the_same_network(net, group):
    sd, norm, scores0, chain0 = net
    scaled = scaled_buffers(group)
    for k in KS:
        v = rescale(sd, group, k)
        _, scores = restate.forward_volume(norm, v, batch_size=2, return_scores=True)
        assert scores.tobytes() == scores0.tobytes(), "%s k=%d: the fp32 scores moved" % (group, k)
        ch = layers.chain(layers.network_input(norm[:1]), v)
        for name, t0 in chain0.items():
            want = t0 * 2.0 ** k if name in scaled else t0
            assert torch.equal(ch[name], want), "%s k=%d: float64 %s is not %s" % (
                group, k, name, "2^k times the original" if name in scaled else "unchanged")
