"""Every forward kernel of the engine in isolation against its float64 reference (oracle/layers.py).

Each check reads the buffers a kernel read, computes the kernel's float64 reference from them and compares the buffers
it wrote element by element with |got - ref| <= tau * 2^-22 * M + floor (M: the same operation on magnitudes).  A
failure names one kernel, and the printed worst element names its slice, pixel and channel.  Also: bit-identity of all
29 buffers across the kernel options that claim it, deep levels with several tiles per CTA, and the float-volume
forward against the oracle.
"""
import time

import numpy as np
import pytest
import torch

from oracle import layers, restate, synth
from test_gpu_probabilities import TOL_P, _expected
from test_layer_reference_host import threshold

pytestmark = pytest.mark.gpu

TOL_MARGIN = 2e-4      # the oracle's top-2 margin below which an fp32 argmax is undecidable (tests/_parity.py)
BN64_ALL_WIDE = sum(1 << i for i in range(1, 18))   # LAYERS 1..17: the tensor-core layers with Cout >= 128
DEFAULTS = {"bn64_mask": 0, "chunk_kb": 1, "chunk_kb_wide": 2, "conv64_cm": 1, "weight_mcast": 0}


def _blob(sd):
    from lungmask_b200.mask import NativeModel
    return NativeModel(sd)


def _load(eng, sd):
    m = _blob(sd)
    eng.load_weights(0, m.blob, m.n_classes)


def _restore(eng, sd):
    for key, v in DEFAULTS.items():
        eng.set_option(key, v)
    _load(eng, sd)


@pytest.fixture(scope="module")
def weights():
    return {"k3": synth.random_state_dict(3, seed=13, head_gain=0.3), "k6": synth.random_state_dict(6, seed=16, head_gain=0.3)}


def _resized(eng, S, seed, H=256, W=256):
    resized, _ = eng.preprocess(synth.phantom(S, H, W, seed=seed))
    return resized


class Buffers:
    """The engine's 29 activation buffers after a forward, read on demand as NCHW float64 (optionally some slices)."""

    def __init__(self, eng, n, norm, scores=None, slices=None):
        self.eng, self.n, self.slices = eng, n, slices
        pick = (lambda a: a) if slices is None else (lambda a: a[slices])
        self.cache = {"input": layers.network_input(pick(norm))}
        if scores is not None:
            self.cache["scores"] = torch.from_numpy(pick(scores)).to(torch.float64)

    def __getitem__(self, name):
        if name not in self.cache:
            a = self.eng.read_activation(layers.ACT_ID[name], self.n)
            self.cache[name] = layers.from_engine(a if self.slices is None else a[self.slices])
        return self.cache[name]


def check_kernels(bufs, sd, tag, kernels=layers.KERNELS):
    """Checks `kernels` on `bufs`; the split-plane outputs rounded to fp16 (the outputs without their lo plane) must be
    rejected at no less than the CPU suite's threshold.  -> the head's Ref if the head was checked."""
    head = None
    for k in kernels:
        refs = layers.reference(k, bufs, sd)
        for out, r in refs.items():
            got = bufs[out]
            c = layers.check(got, r)
            line = layers.fmt("%s %s" % (tag, k.name), out, c)
            if out in layers.ACT and layers.ACT[out][2]:
                lost = layers.check(got.to(torch.float16).to(torch.float64), r, only_active=True)
                line += "  fp16 output rejected %.3f" % lost.rejected
                assert lost.rejected >= threshold(k.name, "out_lo"), (tag, k.name, out, lost)
            print(line)
            assert c.worst <= layers.TAU, (tag, k.name, out, c)
        if k.mode == "Head":
            head = refs["scores"]
    return head


def check_labels(labels, head, tag):
    """The engine's argmax equals the reference's wherever the reference's top-2 margin exceeds twice the score bound."""
    top2 = head.value.topk(2, dim=1).values
    bound = (layers.TAU * layers.UNIT * head.M + head.floor).amax(1)
    decided = (top2[:, 0] - top2[:, 1]) > 2 * bound
    want = head.value.argmax(1)
    diff = torch.from_numpy(labels.astype(np.int64)) != want
    print("%s labels: %d differ, %d undecided of %d" % (tag, int(diff.sum()), int((~decided).sum()), diff.numel()))
    assert not bool((diff & decided).any()), tag


CONFIGS = {
    "k3_n3": dict(weights="k3", n=3, seed=41),
    "k6_n4": dict(weights="k6", n=4, seed=42),
    "trained_n2": dict(weights="trained", n=2, seed=43),
    "bn64": dict(weights="k3", n=3, seed=41, options={"bn64_mask": BN64_ALL_WIDE}),
    "chunk_wide4": dict(weights="k3", n=3, seed=41, options={"chunk_kb": 1, "chunk_kb_wide": 4}),
}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_kernel(engine, weights, config):
    cfg = CONFIGS[config]
    if cfg["weights"] == "trained":
        import bench
        sd = bench.get_weights(3, 7)
    else:
        sd = weights[cfg["weights"]]
    t0 = time.time()
    try:
        for key, v in cfg.get("options", {}).items():
            engine.set_option(key, v)
        _load(engine, sd)     # bn64_mask takes effect at lm_load_weights
        resized = _resized(engine, cfg["n"], cfg["seed"])
        labels, scores = engine.forward(0, resized, return_scores=True)
        bufs = Buffers(engine, cfg["n"], restate.normalise(resized), scores)
        t1 = time.time()
        head = check_kernels(bufs, sd, config)
        check_labels(labels, head, config)
        print("%s: GPU + reads %.1f s, CPU references %.1f s" % (config, t1 - t0, time.time() - t1))
    finally:
        _restore(engine, sd)


def test_activation_info_matches_the_table(engine):
    from lungmask_b200 import _native
    import ctypes as C
    for name, (level, ch, split) in layers.ACT.items():
        lv, c, sp = C.c_int(-1), C.c_int(-1), C.c_int(-1)
        assert _native.lib().lm_debug_activation_info(layers.ACT_ID[name], C.byref(lv), C.byref(c), C.byref(sp)) == 0
        assert (lv.value, c.value, sp.value) == (level, ch, split), name


# ---------------------------------------------------------------------------------------------------------------------
# Bit-identity: all 29 buffers, the scores and the labels
# ---------------------------------------------------------------------------------------------------------------------
def _snapshot(eng, n, labels, scores=None):
    snap = {name: eng.read_activation(layers.ACT_ID[name], n).view(np.uint32) for name in layers.ACT}
    snap["labels"] = labels
    if scores is not None:
        snap["scores"] = scores.view(np.uint32)
    return snap


def _same(a, b, what):
    bad = [k for k in a if k in b and not np.array_equal(a[k], b[k])]
    print("%s: %s" % (what, "bit-identical (%d arrays)" % len([k for k in a if k in b]) if not bad else "differ in " + ", ".join(bad)))
    assert not bad, what


def test_bit_identity(engine, weights):
    sd = weights["k3"]
    n = 3
    try:
        _load(engine, sd)
        resized = _resized(engine, n, 41)
        base = _snapshot(engine, n, *engine.forward(0, resized, return_scores=True))
        _same(base, _snapshot(engine, n, *engine.forward(0, resized, return_scores=True)), "repeat")
        engine.set_option("bn64_mask", BN64_ALL_WIDE)
        _load(engine, sd)
        _same(base, _snapshot(engine, n, *engine.forward(0, resized, return_scores=True)), "bn64_mask (every Cout >= 128 layer)")
        _restore(engine, sd)
        engine.set_option("conv64_cm", 0)
        _same(base, _snapshot(engine, n, *engine.forward(0, resized, return_scores=True)), "conv64_cm = 0")
        engine.set_option("conv64_cm", 1)
        engine.set_option("weight_mcast", 2)
        _same(base, _snapshot(engine, n, *engine.forward(0, resized, return_scores=True)), "weight_mcast = 2")
        engine.set_option("weight_mcast", 0)
        # without a score tap the forward is a CUDA graph: the first call captures it, the second replays it
        captured = _snapshot(engine, n, engine.forward(0, resized))
        replayed = _snapshot(engine, n, engine.forward(0, resized))
        _same(captured, replayed, "graph capture / replay")
        _same(base, captured, "graph / plain launches")
    finally:
        _restore(engine, sd)


# ---------------------------------------------------------------------------------------------------------------------
# Deep levels: a 33-slice wave runs several tiles per CTA at levels 2-4
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine33():
    from lungmask_b200 import _native
    eng = _native.Engine(device=0, batch_capacity=33)
    yield eng
    eng.close()


def test_deep_levels_full_wave(engine33, weights):
    sd = weights["k3"]
    _load(engine33, sd)
    resized = _resized(engine33, 35, 44)
    labels, scores = engine33.forward(0, resized[:33], return_scores=True)
    norm = restate.normalise(resized)
    deep = [k for k in layers.KERNELS if layers.level_of(k) >= 2]
    shallow = [k for k in layers.KERNELS if layers.level_of(k) < 2]
    t0 = time.time()
    check_kernels(Buffers(engine33, 33, norm[:33], scores), sd, "n=33", deep)
    few = [0, 16, 32]
    head = check_kernels(Buffers(engine33, 33, norm[:33], scores, slices=few), sd, "n=33 slices 0/16/32", shallow)
    check_labels(labels[few], head, "n=33")
    # 35 slices = a wave of 33 and a tail wave of 2, which leaves slices 33-34 in the buffers' first two places
    labels, scores = engine33.forward(0, resized, return_scores=True)
    head = check_kernels(Buffers(engine33, 2, norm[33:], scores[33:]), sd, "n=35 tail")
    check_labels(labels[33:], head, "n=35 tail")
    print("deep levels: CPU references %.1f s" % (time.time() - t0))


# ---------------------------------------------------------------------------------------------------------------------
# Float volumes: the float stem in isolation, then scores and labels against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _float_volume(dtype):
    rng = np.random.default_rng(3)
    vol = synth.phantom(4, 200, 216, seed=19).astype(np.float64) + rng.uniform(-0.4, 0.4, size=(4, 200, 216))
    return vol.astype(dtype)


def _index_maps(box):
    (cy, _), (cx, _) = restate.zoom_src_coord(256, box[2] - box[0]), restate.zoom_src_coord(256, box[3] - box[1])
    return np.clip(np.floor(cy + 0.5).astype(np.int64), 0, 255), np.clip(np.floor(cx + 0.5).astype(np.int64), 0, 255)


def _to_voxels(a, boxes, shape, outside):
    """Network-grid maps (S, ..., 256, 256) -> voxels (S, ..., H, W) the way the mask is resampled (utils.reshape_mask),
    `outside` outside each slice's crop box."""
    S, H, W = shape
    out = np.full((S,) + a.shape[1:-2] + (H, W), outside, dtype=a.dtype)
    for s in range(S):
        b = boxes[s]
        iy, ix = _index_maps(b)
        inside = restate.reshape_mask(np.ones((256, 256), np.uint8), b, (H, W)) != 0
        v = np.full(a.shape[1:-2] + (H, W), outside, dtype=a.dtype)
        v[..., b[0]:b[2], b[1]:b[3]] = a[s][..., iy, :][..., ix]
        out[s] = np.where(inside, v, outside)
    return out


def check_float_forward(mask_raw, probs, vol, sd, tag):
    """Scores within TOL_P of the oracle's; every differing mask voxel from a network pixel whose oracle top-2 margin
    is <= TOL_MARGIN.  -> True if no voxel differs."""
    want, _ = _expected(vol, sd)
    err = np.abs(probs - want)
    print("%s: max |dp| vs the oracle %.3e" % (tag, err.max()))
    assert err.max() <= TOL_P, tag
    taps = {}
    restate.inference(vol, sd, batch_size=4, volume_postprocessing=False, taps=taps)
    top2 = np.sort(taps["scores"], axis=1)[:, -2:]
    margin = _to_voxels(top2[:, 1] - top2[:, 0], taps["boxes"], vol.shape, np.inf)
    raw_want = np.asarray([restate.reshape_mask(taps["labels"][i], taps["boxes"][i], vol.shape[1:]) for i in range(vol.shape[0])],
                          dtype=np.uint8)
    diff = mask_raw != raw_want
    print("%s: %d mask voxels differ, largest oracle margin among them %.2e" % (tag, diff.sum(), margin[diff].max() if diff.any() else 0))
    assert np.all(margin[diff] <= TOL_MARGIN), tag
    return not diff.any()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float_volume_kernels_and_scores(engine, weights, dtype):
    sd = weights["k3"]
    _load(engine, sd)
    vol = _float_volume(dtype)
    norm, boxes = engine.preprocess_float(vol)
    tv, _ = restate.preprocess(vol, resolution=[256, 256])
    assert np.array_equal(norm, restate.normalise(tv).astype(np.float32))
    tag = np.dtype(dtype).name
    # the float stem and the other kernels on the buffers of the volume's one wave
    mask_raw = engine.apply_volume_float(0, vol, postprocess=False)
    bufs = Buffers(engine, 4, norm)
    check_kernels(bufs, sd, tag, [k for k in layers.KERNELS if k.mode != "Head"])
    # the head through the probabilities: exp of the reference scores from the engine's C3, resampled like the mask
    mask_p, probs = engine.apply_volume_probs(0, vol, postprocess=False)
    assert np.array_equal(mask_p, mask_raw)
    c3 = layers.from_engine(engine.read_activation(layers.ACT_ID["C3"], 4))
    assert torch.equal(c3, bufs["C3"])
    head = layers.reference(layers.BY_NAME["up_path.3.conv_block.block.3"], {"C3": c3}, sd)["scores"]
    p = head.value.exp()
    tol = p * torch.expm1(layers.TAU * layers.UNIT * head.M + head.floor) + 4 * 2.0 ** -24
    p_vox = _to_voxels(p.numpy(), boxes, vol.shape, 0.0)
    p_vox[:, 0][_to_voxels(np.ones((4, 256, 256)), boxes, vol.shape, 0.0) == 0] = 1.0
    tol_vox = _to_voxels(tol.numpy(), boxes, vol.shape, 0.0)
    over = np.abs(probs.transpose(1, 0, 2, 3) - p_vox) / np.maximum(tol_vox, 1e-300)
    print("%s head via probabilities: worst |dp| / bound %.3f" % (tag, over.max()))
    assert np.all(np.abs(probs.transpose(1, 0, 2, 3) - p_vox) <= tol_vox)
    # scores and labels against the oracle; with no flip the post-processed mask is the oracle's
    if check_float_forward(mask_raw, probs, vol, sd, tag):
        assert np.array_equal(engine.apply_volume_float(0, vol), restate.inference(vol, sd, batch_size=4))


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_half_tensor_volumes(tmp_path, weights, dtype):
    from lungmask_b200 import LMInferer
    sd = weights["k3"]
    p = str(tmp_path / "k3.pth")
    torch.save(sd, p)
    t = torch.from_numpy(_float_volume(np.float32)).to(getattr(torch, dtype)).cuda()
    vol = t.float().cpu().numpy()
    inf = LMInferer(modelpath=p, batch_size=4, volume_postprocessing=False, tqdm_disable=True)
    try:
        mask, probs = inf.apply_with_probabilities(t)
        mask, probs = mask.cpu().numpy(), probs.cpu().numpy()
        assert mask.dtype == np.uint8 and probs.shape == (3,) + vol.shape
        if check_float_forward(mask, probs, vol, sd, dtype):
            want = restate.inference(vol, sd, batch_size=4)
            inf.volume_postprocessing = True
            assert np.array_equal(inf.apply(t).cpu().numpy(), want)
    finally:
        inf.engine.close()
