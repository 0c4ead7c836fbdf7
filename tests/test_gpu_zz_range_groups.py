"""The fp16 range rescue of every activation scale group, bit for bit against the network it rescues.

tests/_range_groups.rescale moves one scale group's activations by 2^k and leaves the network unchanged in fp32
(tests/test_range_groups_host.py).  The BASELINE puts the group's largest value in (32752, 65504], the top octave of fp16;
the VARIANT multiplies the group by a further 2^8m.  Every forward of the variant overflows that group until its scale has
come down by exactly 2^-8m, and then stores the baseline's planes: the epilogue scale sc * 2^k * 2^-k is exact, the
consumers' power-of-two weight normalisation absorbs 2^-k and their in_unscale comes out unchanged.  So the variant must
give the baseline's labels, scores and activations bit for bit, with only that group's scale lowered - no oracle, no
tolerance.  m = 5 exceeds the 2^-32 the engine allows a group and must be refused."""
import numpy as np
import pytest

from _range_groups import GROUPS, rescale, scaled_buffers
from oracle import layers, restate, synth

pytestmark = pytest.mark.gpu

N = 3                     # slices of the per-group forwards
SLOT = 2
TOP = 65504.0
BN64_ALL_WIDE = sum(1 << i for i in range(1, 18))   # LAYERS 1..17: the tensor-core layers with Cout >= 128
DEFAULTS = {"conv64_cm": 1, "bn64_mask": 0, "weight_mcast": 0, "graphs": 1}
SPLIT = [name for name, (_, _, split) in layers.ACT.items() if split]


def _blob(sd):
    from lungmask_b200.mask import NativeModel
    return NativeModel(sd)


def _load(eng, slot, sd):
    m = _blob(sd)
    eng.load_weights(slot, m.blob, m.n_classes)


def _launches(eng):
    return eng.last_timings()["kernel_launches"]


def _scales(eng, slot):
    return {t: eng.activation_scale(slot, layers.ACT_ID[t]) for t in SPLIT}


def _expect_scales(eng, slot, group, m, what):
    got = _scales(eng, slot)
    want = {t: (2.0 ** (-8 * m) if t in GROUPS[group]["tensors"] else 1.0) for t in SPLIT}
    bad = {t: got[t] for t in SPLIT if got[t] != want[t]}
    assert not bad, "%s: scales other than expected (group %s at 2^-%d, every other 1): %s" % (what, group, 8 * m, bad)


def _exponent(mx, lo, hi):
    """The integer a with mx * 2^a in (lo, hi] (lo = hi / 2)."""
    assert mx > 0
    a = int(np.floor(np.log2(hi / mx)))
    while mx * 2.0 ** a > hi:
        a -= 1
    while mx * 2.0 ** (a + 1) <= hi:
        a += 1
    assert lo < mx * 2.0 ** a <= hi
    return a


def _group_max(eng, n):
    return {g: max(float(np.abs(eng.read_activation(layers.ACT_ID[t], n)).max()) for t in spec["tensors"])
            for g, spec in GROUPS.items()}


@pytest.fixture(scope="module")
def weights_path(tmp_path_factory):
    import torch
    import bench
    nets = {"k3": synth.random_state_dict(3, seed=37, head_gain=0.3), "k6": bench.get_weights(6, 8)}
    d = tmp_path_factory.mktemp("range_groups")
    paths = {}
    for name, sd in nets.items():
        paths[name] = str(d / ("%s.pth" % name))
        torch.save(sd, paths[name])
    return nets, paths


@pytest.fixture(scope="module")
def inf(weights_path):
    """An LMInferer of the trained 6-class net; its engine (33 slices per wave) runs every test of this file."""
    from lungmask_b200 import LMInferer
    _, paths = weights_path
    inf = LMInferer(modelpath=paths["k6"], batch_size=20, tqdm_disable=True)
    yield inf
    for k, v in DEFAULTS.items():
        inf.engine.set_option(k, v)


@pytest.fixture(scope="module")
def resized():
    r, _ = restate.preprocess(synth.phantom(N, seed=41), resolution=[256, 256])
    return np.ascontiguousarray(r)


@pytest.fixture(scope="module")
def calib(inf, weights_path, resized):
    """Per net: the scale-1 group maxima on the N slices (no tensor may leave fp16's range at scale 1)."""
    nets, _ = weights_path
    out = {}
    for name, sd in nets.items():
        _load(inf.engine, SLOT, sd)
        inf.engine.forward(SLOT, resized)
        assert all(s == 1.0 for s in _scales(inf.engine, SLOT).values()), "%s overflows at scale 1" % name
        out[name] = _group_max(inf.engine, N)
        print("%s scale-1 group maxima: %s" % (name, ", ".join("%s %.3g" % kv for kv in out[name].items())))
    return out


def _run(eng, slot, resized):
    """labels-only forward (graph path unless graphs = 0), then a forward with scores (individual launches) -> launches of
    each, labels, scores."""
    l0 = _launches(eng)
    labels_first = eng.forward(slot, resized)
    l1 = _launches(eng)
    labels, scores = eng.forward(slot, resized, return_scores=True)
    l2 = _launches(eng)
    return (l1 - l0, l2 - l1), labels_first, labels, scores


def _read_all(eng, n):
    return {t: eng.read_activation(layers.ACT_ID[t], n) for t in layers.ACT}


def _check_group(eng, nets, calib, resized, net, group, ms, read=True):
    sd = nets[net]
    a = _exponent(calib[net][group], TOP / 2, TOP)
    base_sd = rescale(sd, group, a)
    _load(eng, SLOT, base_sd)
    (lb, lb2), bl_first, bl, bs = _run(eng, SLOT, resized)
    assert lb == lb2, "the baseline rescued a tensor"
    _expect_scales(eng, SLOT, group, 0, "%s/%s baseline" % (net, group))
    assert np.array_equal(bl_first, bl)
    bufs = _read_all(eng, N) if read else None
    if read:
        mx = max(float(np.abs(bufs[t]).max()) for t in GROUPS[group]["tensors"])
        assert 256.0 < mx <= TOP, "%s/%s: the baseline's group maximum %.6g is not in (256, 65504]" % (net, group, mx)
    fails = []
    for m in ms:
        what = "%s/%s m=%d" % (net, group, m)
        _load(eng, SLOT, rescale(base_sd, group, 8 * m))
        (lv, lv2), vl_first, vl, vs = _run(eng, SLOT, resized)
        try:
            assert lv == (m + 1) * lb, "%s: %d launches, want %d forwards of %d" % (what, lv, m + 1, lb)
            assert lv2 == lb, "%s: the second call rescued again (%d launches, one forward is %d)" % (what, lv2, lb)
            _expect_scales(eng, SLOT, group, m, what)
            assert np.array_equal(vl_first, bl) and np.array_equal(vl, bl), "%s: labels differ" % what
            assert vs.tobytes() == bs.tobytes(), "%s: scores differ (max |d| %.3g)" % (what, float(np.abs(vs - bs).max()))
            if read:
                down = np.float32(2.0 ** (-8 * m))
                scaled = scaled_buffers(group)
                for t, want in bufs.items():
                    got = eng.read_activation(layers.ACT_ID[t], N)
                    if t in scaled:
                        got = got * down
                    assert got.tobytes() == want.tobytes(), "%s: buffer %s differs from the baseline's (%d values)" % (
                        what, t, int(np.count_nonzero(got != want)))
        except AssertionError as err:
            fails.append(str(err).split("\n")[0])
    assert not fails, "\n".join(fails)
    return base_sd, bl, bs


@pytest.mark.parametrize("net", ["k3", "k6"])
@pytest.mark.parametrize("group", list(GROUPS))
def test_group_rescue_is_exact(inf, weights_path, calib, resized, net, group):
    """m = 1..4 rounds: the baseline's bits, only the group's scale lowered, no rescue on the next call; m = 5: refused,
    and the baseline loaded afterwards gives its bits again."""
    from lungmask_b200 import _native
    nets, _ = weights_path
    eng = inf.engine
    base_sd, bl, bs = _check_group(eng, nets, calib, resized, net, group, (1, 2, 3, 4))
    _load(eng, SLOT, rescale(base_sd, group, 40))
    with pytest.raises(_native.NativeError, match=r"\(-40\)"):
        eng.forward(SLOT, resized, return_scores=True)
    _load(eng, SLOT, base_sd)
    _expect_scales(eng, SLOT, group, 0, "new weights")
    labels, scores = eng.forward(SLOT, resized, return_scores=True)
    assert np.array_equal(labels, bl) and scores.tobytes() == bs.tobytes(), "the baseline's bits after a refusal"
    _expect_scales(eng, SLOT, group, 0, "baseline after a refusal")


OPTIONS = {"conv64_cm0": {"conv64_cm": 0}, "bn64_all_wide": {"bn64_mask": BN64_ALL_WIDE},
           "weight_mcast2": {"weight_mcast": 2}, "graphs0": {"graphs": 0}}
# every producer epilogue: S0 the BN = 64 / conv_cm64 pool epilogue and the upsample U3, C3 the head-fused conv_cm64
# layer's input, A1 / S1 BN = 128, A2 and B4 the wide layers and B4 the 1x1 cascade
OPTION_GROUPS = ["S0", "C3", "A1", "S1", "A2", "B4"]


@pytest.mark.parametrize("option", list(OPTIONS))
def test_group_rescue_with_options(inf, weights_path, calib, resized, option):
    nets, _ = weights_path
    eng = inf.engine
    try:
        for k, v in OPTIONS[option].items():
            eng.set_option(k, v)
        fails = []
        for group in OPTION_GROUPS:
            try:
                _check_group(eng, nets, calib, resized, "k3", group, (1, 4))
            except AssertionError as err:
                fails.append(str(err))
        assert not fails, "\n".join(fails)
    finally:
        for k, v in DEFAULTS.items():
            eng.set_option(k, v)
        _load(eng, SLOT, nets["k3"])   # bn64_mask takes effect at a load


ENTRY_GROUPS = ["A0", "S2", "E1"]
ENTRY_M = 2


@pytest.fixture(scope="module")
def volume():
    """35 slices: a wave of 33 and a wave of 2."""
    return synth.phantom(35, 180, 200, seed=43)


@pytest.mark.parametrize("group", ENTRY_GROUPS)
def test_group_rescue_entry_points(inf, weights_path, calib, volume, group):
    """Whole-volume calls: apply_volume (two waves), the float32 stem, the probabilities, the fusion with the variant in
    either slot and LMInferer.apply on a CUDA tensor.  The baseline's group maximum sits near 2^12 on the calibration
    slices, so that the maximum over this volume stays inside (256, 65504]."""
    import torch
    nets, _ = weights_path
    eng = inf.engine
    sd = nets["k6"]
    a = _exponent(calib["k6"][group], 2.0 ** 11, 2.0 ** 12)
    base_sd = rescale(sd, group, a)
    var_sd = rescale(base_sd, group, 8 * ENTRY_M)
    vol32 = volume.astype(np.float32)
    tvol = torch.from_numpy(volume).to("cuda:0")

    def run(m):
        out = {"volume": eng.apply_volume(0, volume)}
        _expect_scales(eng, 0, group, m, "%s apply_volume" % group)
        out["float32"] = eng.apply_volume_float(0, vol32)
        out["probs"] = eng.apply_volume_probs(0, volume)
        return out

    _load(eng, 0, base_sd)
    want = run(0)
    want_dev = inf.apply(tvol).cpu().numpy()
    _expect_scales(eng, 0, group, 0, "%s baseline" % group)
    for reload in (True, False):   # the first call rescues; the second starts from the lowered scale
        if reload:
            _load(eng, 0, var_sd)
        got = run(ENTRY_M)
        for key in ("volume", "float32"):
            assert np.array_equal(got[key], want[key]), "%s %s differs" % (group, key)
        assert np.array_equal(got["probs"][0], want["probs"][0]), "%s probs: mask differs" % group
        assert got["probs"][1].tobytes() == want["probs"][1].tobytes(), "%s probs differ" % group
        _expect_scales(eng, 0, group, ENTRY_M, "%s after the entry points" % group)
    _load(eng, 0, var_sd)
    assert np.array_equal(inf.apply(tvol).cpu().numpy(), want_dev), "%s LMInferer.apply on a CUDA tensor" % group
    _expect_scales(eng, 0, group, ENTRY_M, "%s LMInferer.apply" % group)
    # the fusion runs both slots' forwards in one call
    _load(eng, 0, base_sd)
    _load(eng, 1, base_sd)
    fused = eng.apply_fused(0, 1, volume)
    for v_slot in (0, 1):
        _load(eng, 0, var_sd if v_slot == 0 else base_sd)
        _load(eng, 1, var_sd if v_slot == 1 else base_sd)
        assert np.array_equal(eng.apply_fused(0, 1, volume), fused), "%s fusion, variant in slot %d" % (group, v_slot)
        _expect_scales(eng, v_slot, group, ENTRY_M, "%s fusion" % group)
        _expect_scales(eng, 1 - v_slot, group, 0, "%s fusion, the other slot" % group)
    _load(eng, 0, sd)
    _load(eng, 1, sd)
