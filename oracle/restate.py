"""CPU restatement of the lungmask hot path.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Every function cites the reference lines (relative to the reference root) it follows.  Integer /
boolean stages use numpy + scipy.ndimage exactly where the reference does (so that timing this
port on host cores is a fair stand-in for the reference's own force_cpu path); the U-Net forward is
a plain fp32 torch-functional evaluation straight from the state_dict (no nn.Module).

Third-party natives the reference relies on but which are absent here (skimage, fill_voids) are
restated in oracle/standins.py.
"""
import numpy as np
import torch
import torch.nn.functional as F
from scipy import ndimage

from .standins import area_closing, cc_label, chunked, fill_voids_fill, regionprops

HU_MIN, HU_MAX = -1024, 600  # utils.py:45
NET_RES = 256  # mask.py:166


# --------------------------------------------------------------------------------------------
# scipy.ndimage.zoom semantics spelled out (utils.py:68,82,108-110,127).  These two helpers are the
# specification the CUDA resize kernels implement; tests check them against scipy itself.
# --------------------------------------------------------------------------------------------
def zoom_out_len(n_in: int, zoom: float) -> int:
    """Output length scipy picks for one axis: round(n_in * zoom) (python round-half-even)."""
    return int(round(n_in * zoom))


def zoom_src_coord(n_in: int, n_out: int):
    """(coord, inside) for every output index of one axis.

    coord = o * ((n_in-1)/(n_out-1)) evaluated in float64 exactly like that (one division, one
    multiplication).  scipy maps coordinates with mode='constant': a coordinate > n_in-1 is OUTSIDE
    and the whole output sample becomes cval = 0.  Because of float64 rounding the LAST index can
    land one ulp above n_in-1 (e.g. 256 -> 12, 200 or 216 samples), in which case the reference
    really produces a zero last row / column; `inside` carries that quirk."""
    if n_out <= 1:
        return np.zeros(n_out, dtype=np.float64), np.ones(n_out, dtype=bool)
    step = np.float64(n_in - 1) / np.float64(n_out - 1)
    c = np.arange(n_out, dtype=np.float64) * step
    return c, c <= np.float64(n_in - 1)


def zoom_nearest(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """order=0 zoom: nearest source index floor(x + 0.5); samples whose coordinate is outside are 0."""
    H, W = img.shape
    (cy, vy), (cx, vx) = zoom_src_coord(H, out_h), zoom_src_coord(W, out_w)
    iy = np.clip(np.floor(cy + 0.5).astype(np.int64), 0, H - 1)
    ix = np.clip(np.floor(cx + 0.5).astype(np.int64), 0, W - 1)
    out = img[iy][:, ix].copy()
    out[~vy, :] = 0
    out[:, ~vx] = 0
    return out


def zoom_linear_to_int(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """order=1 zoom of an integer image, result cast back to the input dtype.

    Per output pixel scipy accumulates, in float64 and in this order,
        t = ((v00*wy0)*wx0) + ((v01*wy0)*wx1) + ((v10*wy1)*wx0) + ((v11*wy1)*wx1)
    with w?0 = 1 - frac, w?1 = frac, neighbours beyond the edge contributing 0 (mode='constant'),
    then rounds half away from zero: (dtype)(t > 0 ? t + 0.5 : t - 0.5).  Samples whose coordinate
    is outside (see zoom_src_coord) are 0.
    """
    H, W = img.shape
    (ys, vyo), (xs, vxo) = zoom_src_coord(H, out_h), zoom_src_coord(W, out_w)
    y0 = np.floor(ys).astype(np.int64)
    x0 = np.floor(xs).astype(np.int64)
    fy, fx = ys - y0, xs - x0
    wy = (1.0 - fy, fy)
    wx = (1.0 - fx, fx)
    src = img.astype(np.float64)
    t = np.zeros((out_h, out_w), dtype=np.float64)
    for dy in (0, 1):
        yy = y0 + dy
        vy = (yy >= 0) & (yy < H)
        for dx in (0, 1):
            xx = x0 + dx
            vx = (xx >= 0) & (xx < W)
            v = src[np.clip(yy, 0, H - 1)[:, None], np.clip(xx, 0, W - 1)[None, :]]
            v = np.where(vy[:, None] & vx[None, :], v, 0.0)
            t = t + (v * wy[dy][:, None]) * wx[dx][None, :]
    t = np.where(t > 0, t + 0.5, t - 0.5)
    info = np.iinfo(img.dtype)
    out = np.clip(np.trunc(t), info.min, info.max).astype(img.dtype)
    out[~vyo, :] = 0
    out[:, ~vxo] = 0
    return out


# --------------------------------------------------------------------------------------------
# Pre-processing
# --------------------------------------------------------------------------------------------
def simple_bodymask(img: np.ndarray) -> np.ndarray:
    """utils.py:55-82.  Body mask on a 128x128 nearest-neighbour thumbnail:
    threshold > -500 HU -> closing (3x3 cross, zero border) -> fill background not 8-connected to
    the frame -> erode x2 (cross) -> keep the largest 4-connected component (first max) ->
    dilate x2 (cross) -> nearest-neighbour zoom back to the slice's shape."""
    oshape = img.shape
    small = ndimage.zoom(img, 128 / np.asarray(oshape), order=0)  # :68
    m = small > -500  # :58,69
    m = ndimage.binary_closing(m)  # :70
    m = ndimage.binary_fill_holes(m, structure=np.ones((3, 3))).astype(int)  # :71-73
    m = ndimage.binary_erosion(m, iterations=2)  # :74
    lab = cc_label(m.astype(int), connectivity=1)  # :75
    regs = regionprops(lab)  # :76
    if regs:  # :77-80
        keep = int(np.argmax([r.area for r in regs])) + 1
        m = ndimage.binary_dilation(lab == keep, iterations=2)
    else:
        m = lab
    return ndimage.zoom(m, np.asarray(oshape) / 128, order=0)  # :81-82


def crop_and_resize(img: np.ndarray, width: int = 192, height: int = 192):
    """utils.py:85-111.  bbox = bounding box of component #1 of an 8-connected labelling of the
    body mask (full frame if the mask is empty); crop; bilinear zoom to (width, height) keeping the
    input dtype."""
    bmask = simple_bodymask(img)
    regs = regionprops(cc_label(bmask))  # :102
    if regs:
        bbox = np.asarray(regs[0].bbox)  # :103-104
    else:
        bbox = (0, 0, bmask.shape[0], bmask.shape[1])  # :105-106
    crop = img[bbox[0]:bbox[2], bbox[1]:bbox[3]]
    out = ndimage.zoom(crop, np.asarray([width, height]) / np.asarray(crop.shape), order=1)  # :108-110
    return out, bbox


def preprocess(img: np.ndarray, resolution=(192, 192)):
    """utils.py:32-52.  Copy, clip to [-1024, 600] HU in the input dtype, per-slice crop+resize."""
    vol = np.clip(np.copy(img), HU_MIN, HU_MAX)
    slices, boxes = [], []
    for sl in vol:
        s, b = crop_and_resize(sl, width=resolution[0], height=resolution[1])
        slices.append(s)
        boxes.append(b)
    return np.asarray(slices), boxes


def normalise(tvolslices: np.ndarray) -> np.ndarray:
    """mask.py:167-168: clamp at 600 then (x + 1024) / 1624 in float64 (cast to fp32 at :178-182)."""
    t = tvolslices.copy()
    t[t > 600] = 600
    return np.divide((t + 1024), 1624)


def reshape_mask(mask: np.ndarray, tbox, origsize) -> np.ndarray:
    """utils.py:114-129.  Nearest-neighbour zoom of the 256x256 mask to the bbox size, pasted into
    a zero float64 canvas of the original slice size."""
    res = np.zeros(origsize, dtype=np.float64)
    size = [tbox[2] - tbox[0], tbox[3] - tbox[1]]
    res[tbox[0]:tbox[2], tbox[1]:tbox[3]] = ndimage.zoom(mask, size / np.asarray(mask.shape), order=0)
    return res


# --------------------------------------------------------------------------------------------
# U-Net forward (resunet.py:58-70 with the get_model configuration, mask.py:58-65)
# --------------------------------------------------------------------------------------------
def _conv_block(x, sd, p):
    """resunet.py:93-105 (non-residual): [conv3x3 pad1 -> ReLU -> BN(eval)] x 2."""
    for conv, bn in ((0, 2), (3, 5)):
        x = F.conv2d(x, sd[f"{p}.{conv}.weight"], sd[f"{p}.{conv}.bias"], padding=1)
        x = F.relu(x)
        x = F.batch_norm(x, sd[f"{p}.{bn}.running_mean"], sd[f"{p}.{bn}.running_var"],
                         sd[f"{p}.{bn}.weight"], sd[f"{p}.{bn}.bias"], training=False, eps=1e-5)
    return x


def unet_forward(x: torch.Tensor, sd: dict, depth: int = 5, taps: dict = None) -> torch.Tensor:
    """x: (N,1,H,W) fp32 -> log-softmax scores (N,K,H,W).  resunet.py:58-70.
    `taps` (optional) collects block outputs / pooled / upsampled tensors keyed like the engine's parity
    taps (S{i}, P{i}, B4, U{j}, E{j}); U{j} is the reference's `up` = conv1x1(upsample(x))."""
    skips = []
    for i in range(depth):  # encoder, :60-64
        x = _conv_block(x, sd, f"down_path.{i}.block")
        if i != depth - 1:
            skips.append(x)
            if taps is not None:
                taps[f"S{i}"] = x
            x = F.avg_pool2d(x, 2)
            if taps is not None:
                taps[f"P{i}"] = x
        elif taps is not None:
            taps["B4"] = x
    for j in range(depth - 1):  # decoder, :66-67 -> :144-148 (upsample mode, :131-133)
        up = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
        up = F.conv2d(up, sd[f"up_path.{j}.up.1.weight"], sd[f"up_path.{j}.up.1.bias"])
        if taps is not None:
            taps[f"U{j}"] = up
        x = torch.cat([up, skips[-j - 1]], 1)  # padding=True => center_crop is the identity
        x = _conv_block(x, sd, f"up_path.{j}.conv_block.block")
        if taps is not None:
            taps[f"E{j}"] = x
    x = F.conv2d(x, sd["last.weight"], sd["last.bias"])  # :69
    return F.log_softmax(x, dim=1)  # :70


def n_classes_of(sd: dict) -> int:
    """mask.py:56: class count = length of the LAST tensor of the state_dict (last.bias)."""
    return len(list(sd.values())[-1])


def forward_volume(tvol_norm: np.ndarray, sd: dict, batch_size: int, return_scores: bool = False):
    """mask.py:172-187: batches of `batch_size` slices, fp32, argmax over classes (first index wins
    ties) -> uint8 labels."""
    labels, scores = [], []
    with torch.inference_mode():
        for chunk in chunked(tvol_norm, batch_size):
            x = torch.as_tensor(np.asarray(chunk)[:, None, ::], dtype=torch.float32)
            out = unet_forward(x, sd)
            labels.append(torch.max(out, 1)[1].numpy().astype(np.uint8))
            if return_scores:
                scores.append(out.numpy())
    lab = np.concatenate(labels, 0) if labels else np.empty((0, NET_RES, NET_RES), np.uint8)
    if return_scores:
        return lab, np.concatenate(scores, 0)
    return lab


# --------------------------------------------------------------------------------------------
# Post-processing
# --------------------------------------------------------------------------------------------
def bbox_3D(labelmap, margin=2):
    """utils.py:361-387: per-axis extent of the non-zero voxels, grown by `margin`, clipped,
    returned half-open as [a0_lo, a0_hi, a1_lo, a1_hi, ...]."""
    out = []
    nd = labelmap.ndim
    for ax in range(nd):
        hit = np.flatnonzero(np.any(labelmap, axis=tuple(a for a in range(nd) if a != ax)))
        lo = max(int(hit[0]) - margin, 0)
        hi = min(int(hit[-1]) + margin + 1, labelmap.shape[ax])
        out += [lo, hi]
    return np.array(out)


def keep_largest_connected_component(mask: np.ndarray) -> np.ndarray:
    """utils.py:390-404: largest full-connectivity component; np.argsort(...)[-1] => among equal
    areas the LAST (highest id) wins."""
    lab = cc_label(mask)
    areas = np.asarray([r.area for r in regionprops(lab)])
    return lab == (np.argsort(areas)[-1] + 1)


def postprocessing(label_image: np.ndarray, spare=(), skip_below: int = 3, taps: dict = None) -> np.ndarray:
    """utils.py:272-358.

    1. 26-connected components of equal label value (ids in raster order)            :293
    2. regions sorted by area, stable                                                 :298-300
    3. every region that sets a new per-label area record maps to its label           :303-308
    4. in ascending ORIGINAL order, each non-record (or spare-labelled) region with
       area >= skip_below is merged into the neighbour region (6-connected dilation
       ring, inside its margin-2 bbox) holding the most ring voxels; ties -> lowest
       id; candidates exclude 0, itself and ids that appear in `spare` (the
       reference compares region ids against label VALUES here - kept);
       the target's cached area (and the label record if it was the record holder)
       grows by the merged area                                                       :310-339
    5. region -> label lookup, spare labels zeroed                                    :341-342
    6. per label (ascending): largest component, holes filled (single-slice volumes:
       area_closing < 64 px; else 3-D fill of background not 6-connected to the
       border), painted in label order                                                :344-358
    """
    spare = list(spare)
    regionmask = cc_label(label_image)
    if taps is not None:
        taps["regions0"] = regionmask.copy()
    origlabels = np.unique(label_image)
    record = np.zeros((max(origlabels) + 1,), dtype=np.uint32)
    regions = regionprops(regionmask, label_image)
    regions.sort(key=lambda r: r.area)
    order_ids = [r.label for r in regions]
    pos = {rid: i for i, rid in enumerate(order_ids)}  # == regionlabels.index(), O(1)

    to_label = np.zeros((len(order_ids) + 1,), dtype=np.uint8)
    for r in regions:
        v = int(r.max_intensity)
        if r.area > record[v]:
            record[v] = r.area
            to_label[r.label] = v

    for r in regions:
        v = int(r.max_intensity)
        if (r.area < record[v] or v in spare) and r.area >= skip_below:
            bb = bbox_3D(regionmask == r.label)
            sub = regionmask[bb[0]:bb[1], bb[2]:bb[3], bb[4]:bb[5]]
            ring = ndimage.binary_dilation(sub == r.label)
            ids, counts = np.unique(sub[ring], return_counts=True)
            target, best, moved = r.label, 0, 0
            for n, c in zip(ids, counts):
                if n != 0 and n != r.label and c > best and n not in spare:
                    best, target, moved = c, n, r.area
            regionmask[regionmask == r.label] = target
            tgt = regions[pos[target]]
            tv = int(tgt.max_intensity)
            if tgt.area == record[tv]:
                record[tv] += moved
            tgt._cache["area"] += moved

    mapped = to_label[regionmask]
    mapped[np.isin(mapped, spare)] = 0
    if taps is not None:
        taps["regions1"] = regionmask.copy()
        taps["mapped"] = mapped.copy()
    return finish_labels(mapped)


def finish_labels(mapped: np.ndarray) -> np.ndarray:
    """utils.py:344-358, step 6 of `postprocessing`: per label, largest component and holes filled."""
    if mapped.shape[0] == 1:
        def fill(x):
            return area_closing(x[0].astype(int), area_threshold=64)[None, :, :] == 1
    else:
        fill = fill_voids_fill

    out = np.zeros(mapped.shape, dtype=np.uint8)
    for v in np.unique(mapped)[1:]:
        out[fill(keep_largest_connected_component(mapped == v))] = v
    return out


# --------------------------------------------------------------------------------------------
# Whole pipeline (mask.py:141-232), numpy-array inputs only
# --------------------------------------------------------------------------------------------
def inference(volume: np.ndarray, sd: dict, batch_size: int = 20, volume_postprocessing: bool = True,
              taps: dict = None) -> np.ndarray:
    """mask.py:141-210 for numpy input.  `taps` (optional dict) receives the stage outputs."""
    raw = volume.copy()
    tvol, boxes = preprocess(raw, resolution=[NET_RES, NET_RES])
    norm = normalise(tvol)
    if taps is not None:
        labels, scores = forward_volume(norm, sd, batch_size, return_scores=True)
        taps.update(resized=tvol, boxes=np.asarray(boxes), scores=scores, labels=labels)
    else:
        labels = forward_volume(norm, sd, batch_size)
    out = postprocessing(labels) if volume_postprocessing else labels
    if taps is not None:
        taps["post"] = out
    out = np.asarray([reshape_mask(out[i], boxes[i], raw.shape[1:]) for i in range(out.shape[0])], dtype=np.uint8)
    return out.astype(np.uint8)


def fuse_pre(res_l: np.ndarray, res_r: np.ndarray):
    """mask.py:228-230: the array (and spare value) that utils.postprocessing receives at mask.py:232.  Voxels the fill
    model marks as lung but the base model left empty get a spare label; voxels the fill model calls background are
    cleared.  `res_l.max() + 1` is uint8 arithmetic, as in the reference."""
    res_l = res_l.copy()
    spare_value = res_l.max() + 1
    res_l[np.logical_and(res_l == 0, res_r > 0)] = spare_value
    res_l[res_r == 0] = 0
    return res_l, spare_value


def fuse(res_l: np.ndarray, res_r: np.ndarray) -> np.ndarray:
    """mask.py:228-232: fuse_pre, then postprocessing dissolves the spare label into neighbouring lobes."""
    pre, spare_value = fuse_pre(res_l, res_r)
    return postprocessing(pre, spare=[spare_value])


def apply(volume: np.ndarray, sd: dict, fill_sd: dict = None, batch_size: int = 20,
          volume_postprocessing: bool = True) -> np.ndarray:
    """LMInferer.apply, mask.py:212-232."""
    if fill_sd is None:
        return inference(volume, sd, batch_size, volume_postprocessing)
    res_l = inference(volume, sd, batch_size, volume_postprocessing)
    res_r = inference(volume, fill_sd, batch_size, volume_postprocessing)
    return fuse(res_l, res_r)
