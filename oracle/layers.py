"""Float64 reference of every forward kernel on its own, and the per-element bound a kernel's output must meet.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The engine's forward is 26 kernels: the stem (1 -> 64 on CUDA cores), 21 tensor-core convolutions (the last one is
the head) and 4 bilinear upsamples.  `KERNELS` lists them in execution order and mirrors `LAYERS`, `ACT` and `UPS` in
lungmask_b200/csrc/engine.cu.  Given the buffers a kernel read, `reference` returns, for every buffer it writes, the
float64 value and a magnitude bound M of the same shape (the same operation on |inputs| and |weights|).  A kernel
with the operand format of DESIGN §3 (hi + lo * 2^-11, 22 significant bits) is accepted when

    |got - ref| <= TAU * 2^-22 * M + floor

element by element, so an error confined to one tile, one halo column, one 64-channel half or the small values of a
tensor is not hidden by the tensor's largest value.  `emulate` restates the kernels' arithmetic (split operands, the
three exact products, fp32 epilogue, split output) and can drop one plane or product, which is how the CPU suite shows
that the bound accepts the arithmetic and rejects a kernel that loses a plane (tests/test_layer_reference_host.py).

Tensors are NCHW torch float64 on the CPU; the engine's buffers are NHWC (`from_engine`).
"""
from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F

TAU = 4.0
UNIT = 2.0 ** -22   # relative precision of the hi + lo * 2^-11 operand format (DESIGN §3)
# Absolute floor.  A value below fp16's normal range (|x| < 2^-14) keeps an fp16-subnormal hi plane, so the split
# carries an absolute precision of 2^-36 (times 1/s for a tensor at a power-of-two scale s, DESIGN §3) instead of 2^-22
# relative.  2^-26 covers that down to s = 2^-10.  Dropping a lo plane moves a value x by up to 2^-12 * |x|, which
# exceeds 2^-26 for every |x| > 2^-14, so the floor can hide a lost plane only on values below fp16's normal range.
FLOOR = 2.0 ** -26
# fp32 expf / logf and the two subtractions of the head's log-softmax (conv_tc.cu): a few ulps of |score| + 1
SOFTMAX_ULPS = 4 * 2.0 ** -23

# Activation buffers, ids as in engine.cu's `enum Act`: name -> (level, channels, split planes)
ACT = {
    "A0": (0, 64, 1), "S0": (0, 64, 1), "P0": (1, 64, 1), "A1": (1, 128, 1), "S1": (1, 128, 1), "P1": (2, 128, 1),
    "A2": (2, 256, 1), "S2": (2, 256, 1), "P2": (3, 256, 1), "A3": (3, 512, 1), "S3": (3, 512, 1), "P3": (4, 512, 1),
    "A4": (4, 1024, 1), "B4": (4, 1024, 1),
    "L0": (4, 512, 0), "U0": (3, 512, 1), "C0": (3, 512, 1), "E0": (3, 512, 1),
    "L1": (3, 256, 0), "U1": (2, 256, 1), "C1": (2, 256, 1), "E1": (2, 256, 1),
    "L2": (2, 128, 0), "U2": (1, 128, 1), "C2": (1, 128, 1), "E2": (1, 128, 1),
    "L3": (1, 64, 0), "U3": (0, 64, 1), "C3": (0, 64, 1),
}
ACT_ID = {name: i for i, name in enumerate(ACT)}

# One kernel: state-dict prefix of its convolution (None for an upsample), mode, source buffers (src1: the skip tensor
# of the virtual concat [up, bridge]; "input" = the normalised network input) and destinations.
Kernel = namedtuple("Kernel", "name prefix mode src0 src1 dst dst_pool")


def _k(prefix, mode, src0, dst, src1=None, dst_pool=None, name=None):
    return Kernel(name or prefix, prefix, mode, src0, src1, dst, dst_pool)


KERNELS = [
    _k("down_path.0.block.0", "ReluBn", "input", "A0", name="stem"),
    _k("down_path.0.block.3", "ReluBnPool", "A0", "S0", dst_pool="P0"),
    _k("down_path.1.block.0", "ReluBn", "P0", "A1"),
    _k("down_path.1.block.3", "ReluBnPool", "A1", "S1", dst_pool="P1"),
    _k("down_path.2.block.0", "ReluBn", "P1", "A2"),
    _k("down_path.2.block.3", "ReluBnPool", "A2", "S2", dst_pool="P2"),
    _k("down_path.3.block.0", "ReluBn", "P2", "A3"),
    _k("down_path.3.block.3", "ReluBnPool", "A3", "S3", dst_pool="P3"),
    _k("down_path.4.block.0", "ReluBn", "P3", "A4"),
    _k("down_path.4.block.3", "ReluBn", "A4", "B4"),
    _k("up_path.0.up.1", "Linear", "B4", "L0"),
    _k(None, "Upsample", "L0", "U0", name="upsample.0"),
    _k("up_path.0.conv_block.block.0", "ReluBn", "U0", "C0", src1="S3"),
    _k("up_path.0.conv_block.block.3", "ReluBn", "C0", "E0"),
    _k("up_path.1.up.1", "Linear", "E0", "L1"),
    _k(None, "Upsample", "L1", "U1", name="upsample.1"),
    _k("up_path.1.conv_block.block.0", "ReluBn", "U1", "C1", src1="S2"),
    _k("up_path.1.conv_block.block.3", "ReluBn", "C1", "E1"),
    _k("up_path.2.up.1", "Linear", "E1", "L2"),
    _k(None, "Upsample", "L2", "U2", name="upsample.2"),
    _k("up_path.2.conv_block.block.0", "ReluBn", "U2", "C2", src1="S1"),
    _k("up_path.2.conv_block.block.3", "ReluBn", "C2", "E2"),
    _k("up_path.3.up.1", "Linear", "E2", "L3"),
    _k(None, "Upsample", "L3", "U3", name="upsample.3"),
    _k("up_path.3.conv_block.block.0", "ReluBn", "U3", "C3", src1="S0"),
    _k("up_path.3.conv_block.block.3", "Head", "C3", "scores"),
]
BY_NAME = {k.name: k for k in KERNELS}


def level_of(k: Kernel) -> int:
    """Spatial level (resolution 256 >> level) of the kernel's output."""
    return ACT[k.dst][0] if k.dst in ACT else 0


def outputs(k: Kernel):
    return [d for d in (k.dst, k.dst_pool) if d is not None]


def from_engine(a: np.ndarray) -> torch.Tensor:
    """An engine activation buffer (N, H, W, C) float32 -> NCHW float64."""
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.float64).permute(0, 3, 1, 2).contiguous()


# --------------------------------------------------------------------------------------------------------------------
# The float64 reference and its magnitude bound
# --------------------------------------------------------------------------------------------------------------------
Ref = namedtuple("Ref", "value M floor active")


def _w(sd, key):
    return sd[key].detach().to(torch.float64)


def _bn_prefix(prefix):
    head, conv = prefix.rsplit(".", 1)
    return "%s.%d" % (head, int(conv) + 2)


def _fold_bn64(sd, prefix):
    """BatchNorm2d(eval) folded in float64: scale = gamma / sqrt(var + 1e-5), shift = beta - mean * scale."""
    p = _bn_prefix(prefix)
    scale = _w(sd, p + ".weight") / torch.sqrt(_w(sd, p + ".running_var") + 1e-5)
    shift = _w(sd, p + ".bias") - _w(sd, p + ".running_mean") * scale
    return scale[None, :, None, None], shift[None, :, None, None]


def _source(k, inputs):
    x = inputs[k.src0]
    return torch.cat([x, inputs[k.src1]], 1) if k.src1 is not None else x


def _conv(x, w, taps):
    return F.conv2d(x, w, padding=1 if taps == 9 else 0)


def _relu_bn(k, x, sd):
    """-> (ref, M, active) of conv -> ReLU -> BN."""
    w, b = _w(sd, k.prefix + ".weight"), _w(sd, k.prefix + ".bias")[None, :, None, None]
    z = _conv(x, w, 9) + b
    scale, shift = _fold_bn64(sd, k.prefix)
    ref = scale * torch.relu(z) + shift
    M = scale.abs() * (_conv(x.abs(), w.abs(), 9) + b.abs()) + shift.abs()
    return ref, M, z > 0


def reference(k: Kernel, inputs: dict, sd: dict) -> dict:
    """float64 output(s) of kernel `k` from the buffers it reads (`inputs`: name -> NCHW float64) -> {output name: Ref}.

    ReluBn / ReluBnPool: ref = scale * relu(conv(x, w) + b) + shift, M = |scale| * (conv(|x|, |w|) + |b|) + |shift|;
    the pooled copy is avg_pool2d of both.  Linear (1x1): ref = conv + b, M = conv(|x|, |w|) + |b|.  Upsample: the
    bilinear x2 of L and of |L|.  Head: the block's conv + ReLU + BN, the 1x1 to K classes, log_softmax; its bound is
    the per-channel tolerance propagated through the 1x1 (|dlogit_j| <= sum_c |w_jc| tol_c) times 2 (log-softmax is
    2-Lipschitz in the max norm), plus a few fp32 ulps of |score| + 1 for expf / logf.  `active` marks the outputs a
    perturbation of the operands can move (ReLU-active ones; every output of the other modes)."""
    x = _source(k, inputs)
    if k.mode == "Upsample":
        up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
        ref = up(x)
        return {k.dst: Ref(ref, up(x.abs()), FLOOR, torch.ones_like(ref, dtype=torch.bool))}
    if k.mode == "Linear":
        w, b = _w(sd, k.prefix + ".weight"), _w(sd, k.prefix + ".bias")[None, :, None, None]
        ref = _conv(x, w, 1) + b
        return {k.dst: Ref(ref, _conv(x.abs(), w.abs(), 1) + b.abs(), FLOOR, torch.ones_like(ref, dtype=torch.bool))}
    ref, M, active = _relu_bn(k, x, sd)
    if k.mode == "ReluBn":
        return {k.dst: Ref(ref, M, FLOOR, active)}
    if k.mode == "ReluBnPool":
        pooled_active = F.avg_pool2d(active.to(torch.float64), 2) > 0
        return {k.dst: Ref(ref, M, FLOOR, active),
                k.dst_pool: Ref(F.avg_pool2d(ref, 2), F.avg_pool2d(M, 2), FLOOR, pooled_active)}
    assert k.mode == "Head", k.mode
    wl, bl = _w(sd, "last.weight"), _w(sd, "last.bias")
    scores = F.log_softmax(_conv(ref, wl, 1) + bl[None, :, None, None], dim=1)
    aw = wl.abs()
    m = 2 * _conv(M, aw, 1).amax(1, keepdim=True)
    fl = 2 * FLOOR * aw.sum((1, 2, 3)).max() + SOFTMAX_ULPS * (scores.abs() + 1)
    return {"scores": Ref(scores, m.expand_as(scores), fl, torch.ones_like(scores, dtype=torch.bool))}


def network_input(norm) -> torch.Tensor:
    """The stem's input: normalised slices (S, 256, 256) as the engine holds them (fp32) -> (S, 1, 256, 256) float64."""
    return torch.as_tensor(np.asarray(norm, dtype=np.float32)[:, None]).to(torch.float64)


def chain(x: torch.Tensor, sd: dict, as_stored: bool = False) -> dict:
    """All 26 references in execution order from the network input x -> {buffer name: tensor, "scores": ...}.
    as_stored: hold every buffer as the engine stores it (split planes `operand`, the 1x1 outputs fp32) before the next
    kernel reads it, so that each kernel sees inputs it could have been given."""
    bufs = {"input": x}
    for k in KERNELS:
        for name, r in reference(k, bufs, sd).items():
            v = r.value
            if as_stored and name in ACT:
                v = operand(v) if ACT[name][2] else _f32(v)
            bufs[name] = v
    return bufs


# --------------------------------------------------------------------------------------------------------------------
# The check
# --------------------------------------------------------------------------------------------------------------------
Check = namedtuple("Check", "worst at rejected n")


def check(got: torch.Tensor, r: Ref, tau: float = TAU, only_active: bool = False) -> Check:
    """Per-element comparison of `got` with r.value.  worst = max |got - ref| / (2^-22 * M + floor / tau) (so an
    element is accepted iff its ratio <= tau) at `at` = (slice, y, x, channel); rejected = the fraction of elements
    whose ratio exceeds tau (among the ReLU-active ones if `only_active`)."""
    got = got.to(torch.float64)
    ratio = (got - r.value).abs() / (UNIT * r.M + r.floor / tau)
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    flat = int(ratio.argmax())
    n, c, y, x = np.unravel_index(flat, tuple(ratio.shape))
    sel = ratio[r.active] if only_active else ratio.reshape(-1)
    rejected = float((sel > tau).to(torch.float64).mean()) if sel.numel() else 0.0
    return Check(float(ratio.reshape(-1)[flat]), (int(n), int(y), int(x), int(c)), rejected, int(sel.numel()))


def fmt(name, out, c: Check) -> str:
    return "%-32s %-6s worst %7.3f at (n=%d, y=%d, x=%d, c=%d)  above tau %.2e" % (name, out, c.worst, *c.at, c.rejected)


# --------------------------------------------------------------------------------------------------------------------
# Emulation of the kernels' arithmetic, with optional faults
# --------------------------------------------------------------------------------------------------------------------
# x_lo: the input's lo plane is lost (the stem and the upsamples, which read fp32, see their input rounded to fp16);
# w_lo: the weights' lo plane is lost; lo_hi: the act_lo * w_hi product is lost (on the tensor-core layers this is the
# same arithmetic as x_lo, since act_lo * w_lo is never formed); out_lo: the output's lo plane is lost.
FAULTS = ("x_lo", "w_lo", "lo_hi", "out_lo")


def faults_of(k: Kernel):
    """The faults that apply to kernel k."""
    if k.mode == "Upsample":
        return ("x_lo", "out_lo")
    if k.name == "stem":
        return ("x_lo", "w_lo", "out_lo")
    if k.mode in ("Linear", "Head"):
        return ("x_lo", "w_lo", "lo_hi")
    return FAULTS


def _f32(t):
    return t.to(torch.float32).to(torch.float64)


def split(t: torch.Tensor, drop_lo: bool = False):
    """fp32 values -> (hi, lo * 2^-11) planes as float64, the roundings of split_f16 (sm90_ptx.cuh) at scale 1."""
    t32 = t.to(torch.float32)
    if float(t32.abs().max()) > 65504.0:
        raise ValueError("the emulation runs at activation scale 1 (a value leaves fp16's range)")
    hi = t32.to(torch.float16).to(torch.float32)
    lo = ((t32 - hi) * 2048.0).to(torch.float16).to(torch.float64) / 2048.0
    return hi.to(torch.float64), (torch.zeros_like(lo) if drop_lo else lo)


def operand(t: torch.Tensor) -> torch.Tensor:
    """The value a split-plane buffer holds for fp32 / float64 data `t`: hi + lo * 2^-11."""
    hi, lo = split(t)
    return hi + lo


def _weight_planes(w: torch.Tensor, drop_lo: bool):
    """engine.cu load_conv: normalise by a power of two to max |w * ws| in (2^14, 2^15], then split -> (hi, lo, ws)."""
    w32 = w.to(torch.float32)
    wmax, ws = float(w32.abs().max()), 1.0
    if wmax > 0:
        while wmax * ws > 32768.0:
            ws *= 0.5
        while wmax * ws <= 16384.0 and ws < 1.0e30:
            ws *= 2.0
    hi, lo = split(w32 * ws, drop_lo)
    return hi, lo, ws


def _fold_bn32(sd, prefix):
    """engine.cu fold_bn: the BN fold in fp32 as torch's CPU eval path computes it."""
    p = _bn_prefix(prefix)
    g, b, mean, var = (sd[p + s].detach().to(torch.float32) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    alpha = (1.0 / torch.sqrt(var + 1e-5)) * g
    return alpha.to(torch.float64)[None, :, None, None], (b - mean * alpha).to(torch.float64)[None, :, None, None]


def _tc_acc(x, w, taps, fault):
    """The tensor-core sum: hi*hi + (hi*lo + lo*hi) * 2^-11 of the split operands, products exact, one fp32 rounding,
    then * in_unscale (the weights' power of two)."""
    xh, xl = split(x, drop_lo=fault == "x_lo")
    wh, wl, ws = _weight_planes(w, drop_lo=fault == "w_lo")
    s = _conv(xh, wh, taps) + _conv(xh, wl, taps)
    if fault != "lo_hi":
        s = s + _conv(xl, wh, taps)
    return _f32(s) / ws


def emulate(k: Kernel, inputs: dict, sd: dict, fault: str = None) -> dict:
    """What kernel k stores, restated in float64 with fp32 / fp16 roundings where the kernel rounds -> {output: tensor}.
    `inputs` must hold values the engine can hold (`operand` for split-plane buffers, fp32 for the others)."""
    assert fault is None or fault in faults_of(k), (k.name, fault)
    x = _source(k, inputs)
    def store(t):
        hi, lo = split(t, drop_lo=fault == "out_lo")
        return hi + lo

    if k.mode == "Upsample":
        xin = x.to(torch.float16).to(torch.float64) if fault == "x_lo" else x
        return {k.dst: store(_f32(F.interpolate(xin, scale_factor=2, mode="bilinear", align_corners=False)))}
    if k.name == "stem":   # CUDA cores, fp32 operands
        xin = x.to(torch.float16).to(torch.float64) if fault == "x_lo" else x
        w = sd[k.prefix + ".weight"].detach()
        if fault == "w_lo":
            wh, _, ws = _weight_planes(w, drop_lo=True)
            w64 = wh / ws
        else:
            w64 = w.to(torch.float64)
        acc = _f32(_conv(xin, w64, 9))
    else:
        acc = _tc_acc(x, sd[k.prefix + ".weight"].detach(), 1 if k.mode == "Linear" else 9, fault)
    b = sd[k.prefix + ".bias"].detach().to(torch.float64)[None, :, None, None]
    z = _f32(acc + b)
    if k.mode == "Linear":
        return {k.dst: z}
    scale, shift = _fold_bn32(sd, k.prefix)
    y = _f32(_f32(torch.relu(z) * scale) + shift)
    if k.mode == "Head":
        wl, bl = sd["last.weight"].detach().to(torch.float64), sd["last.bias"].detach().to(torch.float64)
        logits = _f32(_conv(y, wl, 1) + bl[None, :, None, None])
        return {"scores": F.log_softmax(logits.to(torch.float32), dim=1).to(torch.float64)}
    out = {k.dst: store(y)}
    if k.mode == "ReluBnPool":
        out[k.dst_pool] = store(_f32(F.avg_pool2d(y, 2)))
    return out
