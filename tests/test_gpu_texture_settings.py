"""PyRadiomics' distances, force2D and weightingNorm settings on the GPU (lm_glcm_offsets_dev, lm_neighbour_offsets_dev,
lm_zone_sizes_plane_dev, LMInferer.texture / wavelet_features / filtered_features; DESIGN §4.18).  Every device matrix
must equal the numpy reference of _texture_settings_ref exactly, and the settings must tie back to the verified default
paths where they coincide."""
import json

import numpy as np
import pytest

from _texture_ref import glrlm_ref
from _texture_settings_ref import glcm_offsets_ref, neighbour_offsets_ref, plane_structure, zones_ref
from lungmask_b200 import texture as tx
from oracle import synth

pytestmark = pytest.mark.gpu

SETS = [(1,), (2,), (3,), (1, 2, 3)]
AXES = [None, 0, 1, 2]


@pytest.fixture(scope="module")
def inf():
    import os
    import tempfile
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=47, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _levels(shape, ng, seed, fill=0.7):
    rng = np.random.default_rng(seed)
    L = rng.integers(1, ng + 1, size=shape).astype(np.uint8)
    L[rng.random(shape) > fill] = 0
    return L


def _dev(L):
    import torch
    return torch.from_numpy(np.ascontiguousarray(L)).to("cuda:0")


def check_level_map(eng, L, ng, alpha=0, sets=SETS, axes=AXES):
    tL = _dev(L)
    for d in sets:
        for a in axes:
            offs = tx.offsets(d, a)
            got = eng.glcm_offsets_dev(tL.data_ptr(), L.shape, ng, offs)
            assert np.array_equal(got, glcm_offsets_ref(L, ng, offs)), (L.shape, ng, d, a)
            for g, w in zip(eng.neighbour_offsets_dev(tL.data_ptr(), L.shape, ng, offs, alpha),
                            neighbour_offsets_ref(L, ng, alpha, offs)):
                assert np.array_equal(g, w), (L.shape, ng, d, a, alpha)
    for a in (0, 1, 2):
        got = tx.zones_from_native(eng.zone_sizes_plane_dev(tL.data_ptr(), L.shape, a))
        assert np.array_equal(got, zones_ref(L, plane_structure(a))), (L.shape, a)


@pytest.mark.parametrize("shape", [(9, 13, 37), (1, 5, 70), (2, 2, 2), (3, 1, 33), (40, 2, 1), (1, 1, 1), (5, 7, 3)])
def test_matrices_equal_the_references(inf, shape):
    check_level_map(inf.engine, _levels(shape, 7, seed=sum(shape)), 7)


@pytest.mark.parametrize("ng,alpha", [(255, 0), (255, 3), (91, 1), (90, 0), (30, 2)])
def test_levels_and_alpha(inf, ng, alpha):
    check_level_map(inf.engine, _levels((6, 21, 45), ng, seed=ng + alpha), ng, alpha)


def test_uniform_roi_filling_the_array(inf):
    check_level_map(inf.engine, np.full((7, 11, 35), 3, np.uint8), 3)


def test_phantom_slab(inf):
    vol = synth.phantom(300, 512, 512, seed=100)[140:146]
    for bw in (25, 10):
        L = np.minimum(tx.levels(vol, bw), 255)   # the whole slab, air and body included
        ng = int(L.max())
        check_level_map(inf.engine, L.astype(np.uint8), ng, 0, sets=[(1,), (1, 2, 3)], axes=[None, 0])


def test_offset_refusals(inf):
    from lungmask_b200._native import NativeError
    L = _dev(_levels((3, 4, 5), 3, seed=1))
    bad = [[(0, 0, 0)], [(-1, 0, 0)], [(0, -1, 1)], [(4, 0, 0)], [(1, 0, 0), (1, 0, 0)], tx.offsets((1, 2, 3)) + ((0, 0, 1),)]
    for offs in bad:
        with pytest.raises(NativeError):
            inf.engine.glcm_offsets_dev(L.data_ptr(), (3, 4, 5), 3, offs)
        with pytest.raises(NativeError):
            inf.engine.neighbour_offsets_dev(L.data_ptr(), (3, 4, 5), 3, offs)
    with pytest.raises(NativeError):
        inf.engine.zone_sizes_plane_dev(L.data_ptr(), (3, 4, 5), 3)
    with pytest.raises(NativeError, match="n_levels"):
        inf.engine.glcm_offsets_dev(L.data_ptr(), (3, 4, 5), 2, tx.OFFSETS)   # level 3 above n_levels


@pytest.fixture(scope="module")
def lungs():
    S, H, W = 12, 64, 72
    vol = synth.phantom(S, H, W, seed=31)
    z, y, x = np.ogrid[:S, :H, :W]
    mask = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        mask[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return vol, mask


def _row_levels(vol, mask, row, bw):
    sel = (mask > 0) if row == "lung" else (mask == row)
    vals = vol[sel]
    low, ng = tx.discretisation(float(vals.min()), float(vals.max()), bw)
    L = np.zeros(vol.shape, np.uint8)
    L[sel] = tx.levels(vals, bw, low)
    return L, ng


@pytest.mark.parametrize("distances,axis,norm", [((1,), None, None), ((1, 2, 3), None, None), ((2,), 0, "infinity"),
                                                 ((1, 3), 1, "euclidean"), ((1,), 2, "manhattan"),
                                                 ((3,), None, "no_weighting")])
def test_texture_with_settings(inf, lungs, distances, axis, norm):
    vol, mask = lungs
    sp = (0.7, 0.7, 2.5)
    res = inf.texture(vol, mask, 25, sp, tx.CLASSES, 1, distances, axis is not None, axis or 0, norm)
    st = tx.Settings(tuple(distances), axis, norm)
    assert res.settings == st
    offs, run_offs = st.offsets(), st.run_offsets()
    for row in (1, 2, "lung"):
        L, ng = _row_levels(vol, mask, row, 25)
        r = res[row]
        U = glcm_offsets_ref(L, ng, offs)
        G, N, A = neighbour_offsets_ref(L, ng, 1, offs)
        P = glrlm_ref(L, ng)[[tx.OFFSETS.index(o) for o in run_offs]]
        struct = np.ones((3, 3, 3), bool) if axis is None else plane_structure(axis)
        assert np.array_equal(r.glcm_counts, U) and np.array_equal(r.gldm_counts, G)
        assert np.array_equal(r.ngtdm_counts, N) and np.array_equal(r.ngtdm_sums, A)
        assert np.array_equal(r.glrlm_runs, tx.runs_from_counts(P))
        assert np.array_equal(r.zones, zones_ref(L, struct))   # zones_ref labels the whole map, not the bounding box
        wg = None if norm is None else tx.weights(offs, norm, sp)
        wr = None if norm is None else tx.weights(run_offs, norm, sp)
        assert json.dumps(r.glcm) == json.dumps(tx.glcm_features(U, ng, wg))
        assert json.dumps(r.glrlm) == json.dumps(tx.glrlm_features(P, wr))
        assert json.dumps(r.gldm) == json.dumps(tx.gldm_features(G))
        assert json.dumps(r.ngtdm) == json.dumps(tx.ngtdm_features(N, A))


def test_explicit_defaults_are_todays_call(inf, lungs):
    vol, mask = lungs
    want = json.dumps(inf.texture(vol, mask, 25, None, tx.CLASSES, 2).to_dict())
    got = inf.texture(vol, mask, 25, None, tx.CLASSES, 2, distances=(1,), force2d=False, force2d_dimension=0,
                      weighting_norm=None)
    assert json.dumps(got.to_dict()) == want
    assert json.dumps(inf.texture(vol, mask, 25, None, tx.CLASSES, 2, force2d_dimension=2).to_dict()) == want


def test_one_slice_ties(inf, lungs):
    vol, mask = lungs
    v, m = vol[6:7], mask[6:7]
    flat = inf.texture(v, m, 25, None, tx.CLASSES)
    plane = inf.texture(v, m, 25, None, tx.CLASSES, force2d=True, force2d_dimension=0)
    for row in (1, 2, "lung"):
        assert json.dumps(flat[row].glcm) == json.dumps(plane[row].glcm)
        assert np.array_equal(flat[row].zones, plane[row].zones)
        assert np.array_equal(flat[row].gldm_counts[:, :9], plane[row].gldm_counts)
        assert not flat[row].gldm_counts[:, 9:].any()
        assert np.array_equal(flat[row].ngtdm_counts[:, :9], plane[row].ngtdm_counts)
        assert np.array_equal(flat[row].ngtdm_sums[:, :9], plane[row].ngtdm_sums)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_force2d_glrlm_is_the_in_plane_rows(inf, lungs, axis):
    vol, mask = lungs
    L, ng = _row_levels(vol, mask, "lung", 25)
    tL = _dev(L)
    full = inf.engine.glrlm_dev(tL.data_ptr(), L.shape, ng)
    rows = [d for d, o in enumerate(tx.OFFSETS) if o[axis] == 0]
    res = inf.texture(vol, mask, 25, None, ("glrlm",), force2d=True, force2d_dimension=axis)
    assert np.array_equal(res["lung"].glrlm_runs, tx.runs_from_counts(full[rows]))


def test_settings_refusals(inf, lungs):
    vol, mask = lungs
    for kw in (dict(distances=(4,)), dict(force2d=True, force2d_dimension=3), dict(weighting_norm="chebyshev"),
               dict(weighting_norm="euclidean")):   # the last: no spacing
        with pytest.raises((TypeError, ValueError)):
            inf.texture(vol, mask, 25, None, tx.CLASSES, **kw)
        with pytest.raises((TypeError, ValueError)):
            inf.wavelet_features(vol, mask, classes=("glcm",), **kw)
        with pytest.raises((TypeError, ValueError)):
            inf.filtered_features(vol, mask, image_types=("square",), classes=("glcm",), **kw)


def _width(img, mask):
    """A bin width that keeps every row of `img` within 200 levels."""
    v = img[mask > 0]
    return max(1, int(np.ceil((float(v.max()) - float(v.min()) + 1) / 200.0)))


def test_wavelet_and_filtered_bands_with_settings(inf, lungs):
    from lungmask_b200 import filters as flt
    from lungmask_b200 import wavelet as wv
    vol, mask = lungs
    sp = (0.7, 0.7, 2.5)
    classes = ("glcm", "glszm", "glrlm", "gldm", "ngtdm")
    kw = dict(distances=(1, 2), force2d=True, force2d_dimension=0, weighting_norm="euclidean")
    bands = wv.swt_host(vol, "coif1")
    widths = {n: _width(b, mask) for n, b in bands.items()}
    res = inf.wavelet_features(vol, mask, bin_width=widths, classes=classes, spacing=sp, **kw)
    for name in ("wavelet-LLH", "wavelet-LLL"):
        want = inf.texture(bands[name], mask, widths[name], sp, classes, **kw)
        assert json.dumps(res[name].texture.to_dict()) == json.dumps(want.to_dict())
    img = flt.filter_host(vol, "square")
    bw = _width(img, mask)
    res = inf.filtered_features(vol, mask, image_types=("square",), bin_width=bw, classes=("glcm", "ngtdm"), spacing=sp,
                                **kw)
    want = inf.texture(img, mask, bw, sp, ("glcm", "ngtdm"), **kw)
    assert json.dumps(res["square"].texture.to_dict()) == json.dumps(want.to_dict())
