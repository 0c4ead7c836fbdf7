"""Stand-ins for the reference's third-party natives that are absent from this image.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The reference (`lungmask/utils.py:5-11`, `mask.py:6-11`) imports
`skimage.measure`, `skimage.morphology`, `fill_voids`, `more_itertools`, `SimpleITK`, `pydicom`
(un-pinned in `requirements.txt:1-9`).  None of them is installed here and there is no network, so
the behaviour used on the hot path is restated below from the packages' documented semantics on
top of numpy / scipy.ndimage, and pinned by the reference's own known-answer tests
(`tests/test_utils.py:73-107,124-159`), which `tests/test_oracle_reference.py` re-runs through
these stand-ins.

Restated symbols and the call sites that define what is needed of them:
  skimage.measure.label        utils.py:75 (connectivity=1), :102, :293, :399
  skimage.measure.regionprops  utils.py:76, :102, :298, :400  (+ the `_cache["area"]` poke at :339)
  skimage.morphology.area_closing  utils.py:346-348 (binary image, area_threshold=64)
  fill_voids.fill              utils.py:352
  more_itertools.chunked       mask.py:174
"""
import sys
import types

import numpy as np
from scipy import ndimage


def cc_label(image, connectivity=None):
    """Connected components of equal-valued, non-zero pixels.

    Semantics of `skimage.measure.label(image, connectivity=connectivity)` with background 0:
    two pixels are connected when they are neighbours (connectivity 1 = faces only ...
    connectivity ndim = full 3^ndim neighbourhood, the default) AND hold the same value.
    Component ids are 1..R in raster order of each component's first pixel.
    """
    image = np.asarray(image)
    if image.dtype == bool:
        image = image.astype(np.uint8)
    nd = image.ndim
    if connectivity is None:
        connectivity = nd
    structure = ndimage.generate_binary_structure(nd, connectivity)
    out = np.zeros(image.shape, dtype=np.int64)
    nxt = 0
    for v in np.unique(image):
        if v == 0:
            continue
        lab, n = ndimage.label(image == v, structure=structure)
        if n:
            lab = lab.astype(np.int64)
            out += np.where(lab > 0, lab + nxt, 0)
            nxt += n
    if nxt == 0:
        return out
    # renumber by first occurrence in raster order
    flat = out.ravel()
    ids, first = np.unique(flat, return_index=True)
    keep = ids > 0
    ids, first = ids[keep], first[keep]
    order = np.argsort(first, kind="stable")
    lut = np.zeros(nxt + 1, dtype=np.int64)
    lut[ids[order]] = np.arange(1, len(ids) + 1)
    return lut[out]


class _Region:
    """The four regionprops attributes the reference touches: label, area, bbox, max_intensity."""

    def __init__(self, label, area, bbox, max_intensity):
        self.label = int(label)
        self.bbox = bbox
        self.max_intensity = max_intensity
        self._cache = {"area": int(area)}  # utils.py:339 mutates r.__dict__["_cache"]["area"]

    @property
    def area(self):
        return self._cache["area"]


def regionprops(label_image, intensity_image=None):
    label_image = np.asarray(label_image)
    n = int(label_image.max()) if label_image.size else 0
    if n == 0:
        return []
    areas = np.bincount(label_image.ravel(), minlength=n + 1)
    slices = ndimage.find_objects(label_image, max_label=n)
    if intensity_image is not None:
        maxi = ndimage.maximum(np.asarray(intensity_image), labels=label_image, index=np.arange(1, n + 1))
    regions = []
    for i, sl in enumerate(slices, start=1):
        if sl is None:
            continue
        bbox = tuple(s.start for s in sl) + tuple(s.stop for s in sl)
        mi = maxi[i - 1] if intensity_image is not None else None
        regions.append(_Region(i, areas[i], bbox, mi))
    return regions


def area_closing(image, area_threshold=64, connectivity=1):
    """Binary case of skimage.morphology.area_closing: every 0-valued component (4-connected for
    connectivity=1) with fewer than `area_threshold` pixels is raised to the surrounding level."""
    image = np.asarray(image)
    zero = image == 0
    structure = ndimage.generate_binary_structure(image.ndim, connectivity)
    lab, n = ndimage.label(zero, structure=structure)
    out = image.copy()
    if n:
        areas = np.bincount(lab.ravel(), minlength=n + 1)
        small = areas < area_threshold
        small[0] = False
        out[small[lab]] = 1
    return out


def fill_voids_fill(mask):
    """fill_voids.fill: set every background voxel that is not 6-connected (4-connected in 2-D) to
    the array border."""
    return ndimage.binary_fill_holes(np.asarray(mask) != 0)


def chunked(iterable, n):
    buf = []
    for x in iterable:
        buf.append(x)
        if len(buf) == n:
            yield buf
            buf = []
    if buf:
        yield buf


def install():
    """Register the stand-in modules in sys.modules (idempotent; real packages win if present)."""
    def have(name):
        try:
            __import__(name)
            return True
        except Exception:
            return False

    if not have("skimage"):
        sk = types.ModuleType("skimage")
        me = types.ModuleType("skimage.measure")
        mo = types.ModuleType("skimage.morphology")
        me.label = cc_label
        me.regionprops = regionprops
        mo.area_closing = area_closing
        sk.measure, sk.morphology = me, mo
        sys.modules.update({"skimage": sk, "skimage.measure": me, "skimage.morphology": mo})
    if not have("fill_voids"):
        fv = types.ModuleType("fill_voids")
        fv.fill = fill_voids_fill
        sys.modules["fill_voids"] = fv
    if not have("more_itertools"):
        mi = types.ModuleType("more_itertools")
        mi.chunked = chunked
        sys.modules["more_itertools"] = mi
    if not have("SimpleITK"):
        st = types.ModuleType("SimpleITK")

        class Image:  # only used in isinstance checks / type hints on the numpy path
            pass

        st.Image = Image
        sys.modules["SimpleITK"] = st
    if not have("pydicom"):
        sys.modules["pydicom"] = types.ModuleType("pydicom")
