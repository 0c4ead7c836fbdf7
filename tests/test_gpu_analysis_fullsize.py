"""Label statistics, LAA cluster sizes and whole-ROI texture matrices at the clinical size (lm_label_stats_dev,
lm_laa_clusters_dev, lm_glcm_dev, lm_zone_sizes_dev, lm_zone_sizes_plane_dev, lm_glrlm_dev, lm_neighbour_counts_dev): a
300x512x512 int16 phantom (78.6 M voxels) with an emphysema field and a consolidation-like block in its lungs, against
the numpy oracles of test_gpu_statistics, test_gpu_clusters, test_gpu_texture, _texture_ref and _texture_settings_ref.

At this size the grid-stride loops of stats.cu, clusters.cu and texture.cu run hundreds of iterations per thread, the
per-block shared counters gather millions of counts before they are flushed, and the overflow paths take many entries
from many rows at once: the list of cluster sizes >= 4096 that both labellings share, GLCM pairs outside the shared
band, runs longer than the shared run range, zones of millions of voxels, label counts far past 2^24.  Every test
asserts that its fixture reaches the paths it is there for.

The oracles see each row cropped to its bounding box (the mask is empty and the level map 0 outside it, so no count
changes) and run in a thread pool, which keeps the whole file to about three minutes and 10 GB of host memory on an
8-core host."""
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import scipy.ndimage as ndi

import test_gpu_clusters as tc
import test_gpu_statistics as ts
import test_gpu_texture as tt
from _texture_ref import glrlm_ref, neighbour_ref
from _texture_settings_ref import plane_structure, zones_ref
from lungmask_b200 import texture as tx
from oracle import synth
from test_gpu_clusters import bullae     # noqa: F401  (fixture of test_engine_reuse)
from test_gpu_texture import lungs       # noqa: F401  (fixture of test_engine_reuse)

pytestmark = pytest.mark.gpu

S, H, W = 300, 512, 512
ALL = tx.CLASSES
LAA_HU, BULLA_HU = -950, -990
# A consolidation-like block of constant HU inside lobe 1, 40 x 180 x 40 voxels.  Below -4 HU: with LAA speckle down to
# -1024 HU the lung row spans at most 255 levels at bin width 4.
BLOCK, BLOCK_HU = (slice(100, 140), slice(166, 346), slice(139, 179)), -60
# A bulla of radius 40 centred on the boundary of lobes 4 and 5, with a 2-voxel rim of parenchyma that keeps every other
# LAA voxel out of its 26-neighbourhood: one cluster of the union, one in each of the two lobes.
CROSS, CROSS_R, RIM = (S // 2, 256, 353), 40, 2
DENSE = 4096             # clusters.cuh kClusterDense: larger clusters and zones go to the overflow list
SMEM_LEVELS = 90         # texture.cu kSmemLevels: GLCM triangles in shared memory up to this many levels
SHORT_RUN_WORDS = 53235  # texture.cu kSmemWords: runs up to min(53235 // (13 Ng), longest axis) in shared memory
SMEM_SLOTS = 12          # stats.cu kSmemSlots: labels whose histograms fit shared memory


def k_short(n_levels, shape):
    """The longest run that lm_glrlm_dev counts in shared memory."""
    return min(SHORT_RUN_WORDS // (13 * n_levels), max(shape))


# ---- the scene -----------------------------------------------------------------------------------------------------------
def phantom_lungs():
    """uint8 (S, H, W): synth.phantom's two -850 HU lung ellipsoids, labels 1 (low x) and 2.  They reach the volume's
    first and last planes."""
    z = np.linspace(-0.8, 0.8, S)[:, None, None]
    y = np.linspace(-1, 1, H)[None, :, None]
    x = np.linspace(-1, 1, W)[None, None, :]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, -0.38), (2, 0.38)):
        m[((x - cx) / 0.28) ** 2 + (y / 0.42) ** 2 + (z / 0.9) ** 2 < 1] = label
    return m


def lobes_of(lungs):
    """Five lobes as in test_gpu_shape.five_lobes: lung 1 split at the middle plane and its second half at the middle
    row, lung 2 split at the middle plane."""
    z, y = np.arange(S)[:, None, None], np.arange(H)[None, :, None]
    lobes = lungs.copy()
    lobes[(lungs == 1) & (z >= S // 2)] = 2
    lobes[(lungs == 1) & (z >= S // 2) & (y >= H // 2)] = 3
    lobes[(lungs == 2) & (z < S // 2)] = 4
    lobes[(lungs == 2) & (z >= S // 2)] = 5
    return lobes


def segments_of(lobes, lungs):
    """18 labels: each lobe cut into craniocaudal thirds of its planes (1..15), the block (16), every 101st lung voxel
    (17) and a single voxel (18)."""
    seg = np.zeros_like(lobes)
    for k, box in enumerate(ndi.find_objects(lobes), 1):
        z0, z1 = box[0].start, box[0].stop
        third = (np.arange(z0, z1) - z0) * 3 // (z1 - z0)
        sub = lobes[z0:z1] == k
        seg[z0:z1][sub] = np.broadcast_to((3 * (k - 1) + 1 + third).astype(np.uint8)[:, None, None], sub.shape)[sub]
    seg[BLOCK] = 16
    seg.flat[np.flatnonzero(lungs)[::101]] = 17
    seg[60, 256, 158] = 18
    return seg


def ball(centre, r, shape=(S, H, W)):
    """(box, boolean ball of radius r within the box) around `centre`, clipped to the volume."""
    box = tuple(slice(max(c - r, 0), min(c + r + 1, n)) for c, n in zip(centre, shape))
    z, y, x = np.ogrid[box]
    return box, (z - centre[0]) ** 2 + (y - centre[1]) ** 2 + (x - centre[2]) ** 2 <= r * r


def bullae_list(rng, lungs):
    """(centre, radius) of the bullae: some against the first and last planes, some across lobe boundaries, and about
    150 of radius 3..16 at random lung voxels, apart from each other, from the block and from the crossing bulla."""
    fixed = [((0, 256, 158), 24), ((S - 1, 256, 353), 30), ((0, 230, 353), 12), ((S - 1, 300, 158), 16),   # faces
             ((S // 2, 200, 205), 12), ((225, 256, 158), 14), ((152, 256, 120), 10)]   # lobes 1|2, 2|3, 1|2|3
    lo = np.array([s.start for s in BLOCK]) - 1
    hi = np.array([s.stop for s in BLOCK])
    placed = list(fixed)
    idx = np.flatnonzero(lungs)
    for c in rng.choice(idx, size=400, replace=False):
        if len(placed) >= len(fixed) + 150:
            break
        c = np.array(np.unravel_index(c, lungs.shape))
        r = int(rng.integers(3, 17))
        if np.all((c + r >= lo) & (c - r <= hi)):   # touches the block
            continue
        if np.linalg.norm(c - CROSS) <= CROSS_R + RIM + r + 1:
            continue
        if any(np.linalg.norm(c - np.array(p)) <= r + q + 1 for p, q in placed):
            continue
        placed.append((tuple(int(v) for v in c), r))
    return placed


def make_scene():
    """{"vol": int16, "volf": float32 copy with +-0.5 jitter and ~1 % NaN, "masks": {name: uint8}, "cross": {row: voxels
    of the crossing bulla in that lobe}}."""
    vol = synth.phantom(S, H, W, seed=100)
    lungs = phantom_lungs()
    lobes = lobes_of(lungs)
    rng = np.random.default_rng(101)
    cbox, cball = ball(CROSS, CROSS_R + RIM)
    rim_values = np.maximum(vol[cbox], LAA_HU + 1)   # the phantom's noise, never LAA
    # emphysema: 3 % LAA speckle of -1024..-951 HU, then -990 HU bullae
    inside = np.flatnonzero(lungs)
    pick = inside[rng.random(inside.size) < 0.03]
    vol.flat[pick] = rng.integers(-1024, LAA_HU, pick.size)
    del inside, pick
    for centre, r in bullae_list(rng, lungs):
        box, b = ball(centre, r)
        vol[box][b & (lungs[box] > 0)] = BULLA_HU
    vol[cbox][cball] = rim_values[cball]
    box, b = ball(CROSS, CROSS_R)
    vol[box][b] = BULLA_HU
    cross = {k: int((b & (lobes[box] == k)).sum()) for k in (4, 5)}
    vol[BLOCK] = BLOCK_HU
    masks = {"lungs": lungs, "lobes": lobes, "segments": segments_of(lobes, lungs), "whole": np.ones(vol.shape, np.uint8)}
    volf = vol.astype(np.float32)
    volf += rng.uniform(-0.5, 0.5, vol.shape).astype(np.float32)
    volf[rng.random(vol.shape) < 0.01] = np.nan
    return {"vol": vol, "volf": volf, "masks": masks, "cross": cross}


def boxes(mask):
    """{row: bounding box} of every label value in the mask and of "lung" (mask > 0)."""
    out = {k: b for k, b in enumerate(ndi.find_objects(mask), 1) if b is not None}
    out["lung"] = tuple(slice(min(b[a].start for b in out.values()), max(b[a].stop for b in out.values())) for a in range(3))
    return out


def crop(vol, mask):
    """The volume and the mask within the mask's bounding box."""
    box = boxes(mask)["lung"]
    return vol[box], mask[box]


# ---- references: the existing oracles, run in a thread pool (scipy.ndimage.label and the large numpy operations release
# the GIL), the largest jobs first -------------------------------------------------------------------------------------------
def statistics_references(pool, scene):
    """{(mask name, dtype name): test_gpu_statistics.oracle} for the four masks and the int16 / float32 volumes.  The
    cropped cases run in the pool; the two whole-volume ones after them, one at a time (each holds about 2.5 GB of
    float64 copies)."""
    vols = {"int16": scene["vol"], "float32": scene["volf"]}

    def oracle(case):
        return ts.oracle(*crop(vols[case[1]], scene["masks"][case[0]]))
    cases = [(m, d) for m in ("segments", "lobes", "lungs") for d in vols]
    want = dict(zip(cases, pool.map(oracle, cases)))
    want.update({("whole", d): oracle(("whole", d)) for d in vols})
    return want


CLUSTER_CASES = (("lobes", 26), ("lobes", 6), ("lobes", 4), ("lungs", 26), ("lungs", 6))


def cluster_references(pool, scene):
    """{(mask name, connectivity): test_gpu_clusters.oracle at -950 HU}."""
    vol, masks = scene["vol"], scene["masks"]
    return dict(zip(CLUSTER_CASES, pool.map(lambda c: tc.oracle(*crop(vol, masks[c[0]]), LAA_HU, c[1]), CLUSTER_CASES)))


def row_levels(vol, mask, bw):
    """{row: (level map of the row's box, voxels, low, ng)} through test_gpu_texture.ref_levels, largest box first."""
    out = {}
    for row, box in sorted(boxes(mask).items(), key=lambda kv: -np.prod([s.stop - s.start for s in kv[1]])):
        m = mask[box]
        out[row] = tt.ref_levels(vol[box], m > 0 if row == "lung" else m == row, bw)
    return out


def texture_references(pool, vol, mask, bw):
    """{row: (voxels, low, ng, U, zones, runs, (G, N, A))}: test_gpu_texture.ref_matrices, _texture_ref.glrlm_ref and
    neighbour_ref (alpha 0) of every row's cropped level map; runs padded to the device's length axis max(vol.shape)."""
    levels = row_levels(vol, mask, bw)
    jobs = {row: (pool.submit(tt.ref_matrices, L, ng), pool.submit(glrlm_ref, L, ng), pool.submit(neighbour_ref, L, ng, 0))
            for row, (L, n, low, ng) in levels.items()}
    out = {}
    for row, (matrices, runs, neighbours) in jobs.items():
        _, n, low, ng = levels[row]
        P = runs.result()
        P = np.pad(P, ((0, 0), (0, 0), (0, max(vol.shape) - P.shape[2])))
        out[row] = (n, low, ng) + matrices.result() + (P, neighbours.result())
    return out


def plane_zone_references(pool, vol, mask, bw):
    """{axis: {row: (voxels, low, ng, zones)}}: _texture_settings_ref.zones_ref with plane_structure(axis) of every row's
    cropped level map, for the axes 0, 1 and 2."""
    levels = row_levels(vol, mask, bw)
    jobs = {a: {row: pool.submit(zones_ref, L, plane_structure(a)) for row, (L, _, _, _) in levels.items()} for a in range(3)}
    return {a: {row: levels[row][1:] + (f.result(),) for row, f in rows.items()} for a, rows in jobs.items()}


# ---- tests ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene():
    return make_scene()


@pytest.fixture(scope="module")
def pool():
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as p:
        yield p


@pytest.fixture(scope="module")
def inf():
    import tempfile
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=45, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def test_label_statistics(inf, scene, pool):
    """statistics() with test_gpu_statistics' percentiles and thresholds on the lung, lobe, 18-segment and whole-volume
    masks, int16 and float32 with NaN: the 18 labels take the global-histogram path, the whole-volume rows count
    78.6 M voxels."""
    want = statistics_references(pool, scene)
    vols = {"int16": _cuda(scene["vol"]), "float32": _cuda(scene["volf"])}
    for name, m in scene["masks"].items():
        tm = _cuda(m)
        for dtype, tv in vols.items():
            got = inf.statistics(tv, tm, percentiles=ts.Q, thresholds=ts.T)
            ts.check(got, want[name, dtype])
    assert len(want["segments", "int16"]) == 18 + 1 > SMEM_SLOTS
    assert want["whole", "int16"][1]["voxels"] == S * H * W > 2 ** 24
    assert want["whole", "float32"]["lung"]["nan_voxels"] > 2 ** 19


def test_laa_clusters(inf, scene, pool):
    """laa_clusters() at -950 HU on the lung and lobe masks, 26- and 6-connected, and 4-connected on the lobes: every
    row's (size, count) pairs.  The speckle gives more than 10^5 clusters, the bullae many clusters of 4096 voxels or
    more in several rows (the overflow list both labellings share), and the crossing bulla is one cluster of the union
    and of lung 2, and one in each of lobes 4 and 5."""
    want = cluster_references(pool, scene)
    tv = _cuda(scene["vol"])
    cross = scene["cross"]
    for name, conn in CLUSTER_CASES:
        res = inf.laa_clusters(tv, _cuda(scene["masks"][name]), connectivity=conn)
        tc.check(res, want[name, conn])
        assert res["lung"].clusters > 100_000, (name, conn)
        rows = (1, 2, 3, 4, 5) if name == "lobes" else (1, 2)
        big = {r: int(res[r].counts[res[r].sizes >= DENSE].sum()) for r in rows + ("lung",)}
        if conn == 4:   # in-plane: only the crossing bulla's middle planes hold discs of 4096 voxels or more
            assert big["lung"] == big[4] + big[5] > 0, big
            continue
        assert big["lung"] >= 50 and sum(big[r] > 0 for r in rows) >= min(3, len(rows)), (name, conn, big)
        assert res["lung"].largest_voxels == cross[4] + cross[5]
        if name == "lobes":
            assert (res[4].largest_voxels, res[5].largest_voxels) == (cross[4], cross[5])
        else:
            assert res[2].largest_voxels == cross[4] + cross[5]


def _classes_json(row, classes):
    return json.dumps({c: getattr(row, c) for c in classes})   # NaN-safe, bit-exact through repr


@pytest.mark.parametrize("bw", [25, 4, 200])
def test_texture_matrices(inf, scene, pool, bw):
    """texture() with all five classes on the lobe mask.  25: the realistic case, 39 levels; 4: 242 levels in lobe 1 and
    the lung row, so the GLCM counts the band j - i < 16 in shared memory and the rest with global atomics; 200: zones of
    millions of voxels.  The block's runs of 180 voxels are longer than the shared run range at 25 and 4; at 200 the lung
    row has 6 levels, the shared range (53235 // 78) is capped at the longest axis, and no run can exceed it."""
    vol, lobes = scene["vol"], scene["masks"]["lobes"]
    res = inf.texture(_cuda(vol), _cuda(lobes), bin_width=bw, classes=ALL)
    want = texture_references(pool, vol, lobes, bw)
    tt.check(res, {row: (None,) + w[:5] for row, w in want.items()}, bw)
    for row, (n, low, ng, U, zones, P, neighbours) in want.items():
        r = res[row]
        np.testing.assert_array_equal(r.glrlm_runs, tx.runs_from_counts(P), err_msg=str(row))
        for got, ref in zip((r.gldm_counts, r.ngtdm_counts, r.ngtdm_sums), neighbours):
            np.testing.assert_array_equal(got, ref, err_msg=str(row))
        expect = tx.build_row(256 if row == "lung" else row, r.name, n, bw, low, ng, U, zones, ALL, P, neighbours)
        assert _classes_json(r, ALL) == _classes_json(expect, ALL), row
    lung = res["lung"]
    ng = lung.n_levels
    assert lung.zones[:, 1].max() >= DENSE
    if bw == 200:
        assert k_short(ng, vol.shape) == max(vol.shape) and lung.zones[:, 1].max() > 10 ** 6
    else:
        assert lung.glrlm_runs[:, 2].max() > k_short(ng, vol.shape), (bw, ng)
    if bw == 4:
        iu, ju = np.triu_indices(ng)
        assert ng > SMEM_LEVELS and res[1].n_levels > SMEM_LEVELS
        assert lung.glcm_counts[:, ju - iu >= 16].sum() > 0   # pairs outside the shared band
    else:
        assert ng <= SMEM_LEVELS


def test_force2d_zones(inf, scene, pool):
    """texture(classes=("glszm",), force2d=True) on the lobe mask at bin width 25 for force2d_dimension 0, 1 and 2
    (lm_zone_sizes_plane_dev): the 8-connected in-plane zones of every row and their features."""
    vol, lobes = scene["vol"], scene["masks"]["lobes"]
    want = plane_zone_references(pool, vol, lobes, 25)
    tv, tm = _cuda(vol), _cuda(lobes)
    for axis in (0, 1, 2):
        res = inf.texture(tv, tm, bin_width=25, classes=("glszm",), force2d=True, force2d_dimension=axis)
        for row, (n, low, ng, zones) in want[axis].items():
            r = res[row]
            assert (r.voxels, r.low, r.n_levels) == (n, low, ng), (axis, row)
            np.testing.assert_array_equal(r.zones, zones, err_msg="axis %d row %s" % (axis, row))
            expect = tx.build_row(256 if row == "lung" else row, r.name, n, 25, low, ng, zones=zones, classes=("glszm",))
            assert _classes_json(r, ("glszm",)) == _classes_json(expect, ("glszm",)), (axis, row)
        assert res["lung"].zones[:, 1].max() >= DENSE, axis


def test_engine_reuse(inf, lungs, bullae):
    """After the full-size calls the engine's work areas are at their largest: the small texture and cluster cases of
    test_gpu_texture, test_gpu_texture_classes and test_gpu_clusters on the same LMInferer read no stale counters."""
    import test_gpu_texture_classes as ttc
    vol, mask, lobes = lungs
    for m in (mask, lobes):
        tt.check(inf.texture(vol, m), tt.reference(vol, m, 25), 25)
        ttc.check(inf.texture(vol, m, classes=ALL), vol, m, 25)
    bvol, bmask = bullae
    for conn in tc.CONNS:
        tc.check(inf.laa_clusters(bvol, bmask, connectivity=conn), tc.oracle(bvol, bmask, LAA_HU, conn))
