"""PyRadiomics' distances, force2D and weightingNorm settings of the texture matrices (DESIGN §4.18), on the CPU:
texture.offsets against a literal restatement of the rule, the numpy references of _texture_settings_ref against
voxel-by-voxel loops and per-plane labelling, the weights and the weighted merge against a literal restatement, and the
argument checks, to_dict keys and CLI checks."""
import itertools
import json
import math

import numpy as np
import pytest

from _texture_settings_ref import glcm_offsets_ref, neighbour_offsets_ref, plane_structure, zones_ref
from lungmask_b200 import texture as tx

SETS = [(1,), (2,), (3,), (1, 2, 3)]
AXES = [None, 0, 1, 2]


def literal_offsets(distances, axis):
    out = []
    for dz in range(-3, 4):
        for dy in range(-3, 4):
            for dx in range(-3, 4):
                o = (dz, dy, dx)
                if max(abs(dz), abs(dy), abs(dx)) not in distances:
                    continue
                first = [c for c in o if c != 0][0]
                if first <= 0:
                    continue
                if axis is not None and o[axis] != 0:
                    continue
                out.append(o)
    return tuple(out)


@pytest.mark.parametrize("distances", SETS + [(3, 1, 1), (2, 3)])
@pytest.mark.parametrize("axis", AXES)
def test_offsets_follow_the_rule(distances, axis):
    got = tx.offsets(distances, axis)
    assert got == literal_offsets(set(distances), axis)
    assert list(got) == sorted(got) and len(set(got)) == len(got)


def test_offset_set_sizes_and_default():
    assert [len(tx.offsets(d)) for d in SETS] == [13, 49, 109, 171]
    for a in (0, 1, 2):
        assert [len(tx.offsets(d, a)) for d in SETS] == [4, 8, 12, 24]
    assert tx.offsets() == tx.OFFSETS == tx.offsets((1,), None)
    assert tx.Settings().offsets() == tx.OFFSETS and tx.Settings().run_offsets() == tx.OFFSETS
    for a in (0, 1, 2):
        run = tx.Settings((1, 2), a).run_offsets()
        assert run == tuple(o for o in tx.OFFSETS if o[a] == 0) and len(run) == 4


def _levels(shape, ng, seed, fill=0.7):
    rng = np.random.default_rng(seed)
    L = rng.integers(1, ng + 1, size=shape).astype(np.uint8)
    L[rng.random(shape) > fill] = 0
    return L


def loop_glcm(L, ng, offs):
    T = ng * (ng + 1) // 2
    U = np.zeros((len(offs), T), np.int64)
    n0, n1, n2 = L.shape
    for d, (dz, dy, dx) in enumerate(offs):
        for z, y, x in itertools.product(range(n0), range(n1), range(n2)):
            zz, yy, xx = z + dz, y + dy, x + dx
            if not (0 <= zz < n0 and 0 <= yy < n1 and 0 <= xx < n2):
                continue
            a, b = int(L[z, y, x]), int(L[zz, yy, xx])
            if a and b:
                i, j = min(a, b), max(a, b)
                U[d, (i - 1) * ng - (i - 1) * (i - 2) // 2 + (j - i)] += 1
    return U


def loop_neighbours(L, ng, alpha, offs):
    cols = 2 * len(offs) + 1
    G, N, A = (np.zeros((ng, cols), np.int64) for _ in range(3))
    n0, n1, n2 = L.shape
    for z, y, x in itertools.product(range(n0), range(n1), range(n2)):
        a = int(L[z, y, x])
        if not a:
            continue
        w = s = c = 0
        for o in offs:
            for sgn in (1, -1):
                zz, yy, xx = z + sgn * o[0], y + sgn * o[1], x + sgn * o[2]
                if 0 <= zz < n0 and 0 <= yy < n1 and 0 <= xx < n2 and L[zz, yy, xx]:
                    b = int(L[zz, yy, xx])
                    w += 1
                    s += b
                    c += abs(b - a) <= alpha
        G[a - 1, c] += 1
        N[a - 1, w] += 1
        A[a - 1, w] += abs(w * a - s)
    return G, N, A


@pytest.mark.parametrize("shape", [(5, 6, 7), (1, 4, 9), (2, 2, 3), (7, 3, 1)])
@pytest.mark.parametrize("distances,axis", [((1,), None), ((2,), 0), ((3,), None), ((1, 2, 3), 1), ((1, 3), 2)])
def test_references_against_voxel_loops(shape, distances, axis):
    ng = 5
    L = _levels(shape, ng, seed=sum(shape) + len(distances))
    offs = tx.offsets(distances, axis)
    assert np.array_equal(glcm_offsets_ref(L, ng, offs), loop_glcm(L, ng, offs))
    for alpha in (0, 1):
        for got, want in zip(neighbour_offsets_ref(L, ng, alpha, offs), loop_neighbours(L, ng, alpha, offs)):
            assert np.array_equal(got, want)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_plane_zones_against_per_plane_labelling(axis):
    import scipy.ndimage as ndi
    L = _levels((6, 7, 8), 3, seed=axis, fill=0.8)
    want = {}
    for k in range(L.shape[axis]):
        plane = np.take(L, k, axis=axis)
        for lv in range(1, 4):
            lab, n = ndi.label(plane == lv, np.ones((3, 3), bool))
            for size in np.bincount(lab.ravel())[1:]:
                want[(lv, int(size))] = want.get((lv, int(size)), 0) + 1
    got = zones_ref(L, plane_structure(axis))
    assert {(int(a), int(b)): int(c) for a, b, c in got} == want
    one = L[:1]
    assert np.array_equal(zones_ref(one, plane_structure(0)), zones_ref(one, np.ones((3, 3, 3), bool)))


def literal_weight(o, norm, spacing_xyz):
    s = (spacing_xyz[2], spacing_xyz[1], spacing_xyz[0])
    d = [abs(o[k]) * s[k] for k in range(3)]
    if norm == "infinity":
        return math.exp(-max(d) ** 2)
    if norm == "euclidean":
        return math.exp(-sum(x * x for x in d))
    if norm == "manhattan":
        return math.exp(-sum(d) ** 2)
    return 1.0


@pytest.mark.parametrize("norm", tx.WEIGHTING_NORMS)
def test_weights_restate_the_norms(norm):
    sp = (0.7, 0.8, 2.5)
    offs = tx.offsets((1, 2, 3))
    w = tx.weights(offs, norm, sp)
    assert w.dtype == np.float64 and w.shape == (len(offs),)
    for o, x in zip(offs, w):
        assert x == pytest.approx(literal_weight(o, norm, sp), rel=1e-12, abs=0)   # summation order
    with pytest.raises(ValueError):
        tx.weights(offs, "chebyshev", sp)


@pytest.mark.parametrize("norm", tx.WEIGHTING_NORMS)
def test_weighted_merge_is_one_matrix(norm):
    ng = 6
    L = _levels((4, 9, 10), ng, seed=3)
    sp = (0.6, 0.6, 1.5)
    offs = tx.offsets((1, 2), None)
    U = glcm_offsets_ref(L, ng, offs)
    w = tx.weights(offs, norm, sp)
    iu, ju = np.triu_indices(ng)
    M = np.zeros((ng, ng))
    for o, u in enumerate(U):
        P = np.zeros((ng, ng))
        P[iu, ju] += u
        P[ju, iu] += u
        M += w[o] * P
    assert tx.glcm_features(U, ng, w) == tx._glcm_direction(M, ng)
    runs = np.zeros((4, ng, 5), np.int64)
    runs[0, 1, 0], runs[1, 2, 3], runs[3, 5, 4] = 7, 2, 1
    rw = tx.weights(tx.offsets((1,), 0), norm, sp)
    R = sum(rw[d] * runs[d] for d in range(4))
    i, k = np.nonzero(R)
    f = tx.glszm_features(i + 1, k + 1, R[i, k], float(np.sum((k + 1) * R[i, k])))
    assert tx.glrlm_features(runs, rw) == dict(zip(tx.GLRLM_FEATURES, (f[g] for g in tx.GLSZM_FEATURES)))
    assert all(math.isnan(v) for v in tx.glcm_features(np.zeros_like(U), ng, w).values())
    assert all(math.isnan(v) for v in tx.glrlm_features(np.zeros_like(runs), rw).values())


def test_wider_neighbour_matrices_use_their_columns():
    ng = 4
    L = _levels((5, 6, 7), ng, seed=9)
    offs = tx.offsets((1, 2))
    G, N, A = neighbour_offsets_ref(L, ng, 0, offs)
    assert G.shape == (ng, 125)   # K = 2 (13 + 49)
    i, c = np.nonzero(G)
    f = tx.glszm_features(i + 1, c + 1, G[i, c], int(G.sum()))
    assert tx.gldm_features(G)["LargeDependenceEmphasis"] == f["LargeAreaEmphasis"]
    n = tx.ngtdm_features(N, A)
    keep = np.nonzero(N[:, 1:].sum(axis=1))[0]
    s = [math.fsum(float(A[l, w]) / w for w in range(1, 125)) for l in keep]
    p = N[keep, 1:].sum(axis=1) / float(N[:, 1:].sum())
    assert n["Coarseness"] == 1.0 / np.sum(p * np.array(s))


@pytest.mark.parametrize("kwargs,exc", [
    (dict(distances=()), ValueError), (dict(distances=(0,)), ValueError), (dict(distances=(4,)), ValueError),
    (dict(distances="1"), TypeError), (dict(distances=1), TypeError), (dict(distances=(1.0,)), TypeError),
    (dict(distances=(True,)), TypeError), (dict(force2d=1), TypeError), (dict(force2d_dimension=3), ValueError),
    (dict(force2d=True, force2d_dimension=-1), ValueError), (dict(force2d_dimension=1.0), TypeError),
    (dict(weighting_norm="chebyshev"), ValueError), (dict(weighting_norm="Euclidean"), ValueError)])
def test_settings_refusals(kwargs, exc):
    with pytest.raises(exc):
        tx.check_settings(**kwargs)


def test_settings_values():
    assert tx.check_settings() == tx.Settings()
    assert tx.check_settings(distances=[3, 1, 1]) == tx.Settings((1, 3))
    assert tx.check_settings(force2d=False, force2d_dimension=2) == tx.Settings()
    assert tx.check_settings(force2d=True, force2d_dimension=2) == tx.Settings((1,), 2)
    tx.check_weighting_spacing(tx.Settings(weighting_norm="no_weighting"), None)
    tx.check_weighting_spacing(tx.Settings(weighting_norm="infinity"), (1.0, 1.0, 1.0))
    with pytest.raises(ValueError, match="spacing"):
        tx.check_weighting_spacing(tx.Settings(weighting_norm="manhattan"), None)


def _features(settings):
    row = tx.build_row(1, "right lung", 0, 25, classes=tx.CLASSES, columns=2 * len(settings.offsets()) + 1)
    return tx.TextureFeatures((1.0, 1.0, 2.0), 25, [row], tx.CLASSES, 0, settings)


def test_to_dict_keys():
    base = _features(tx.Settings()).to_dict()
    assert not {"distances", "force2d_dimension", "weighting_norm", "offsets"} & set(base)
    assert json.dumps(base) == json.dumps(tx.TextureFeatures((1.0, 1.0, 2.0), 25, _features(tx.Settings()).rows,
                                                             tx.CLASSES, 0).to_dict())
    d = _features(tx.Settings((1, 2), 0, "euclidean")).to_dict()
    assert d["distances"] == [1, 2] and d["force2d_dimension"] == 0 and d["weighting_norm"] == "euclidean"
    assert d["offsets"] == [list(o) for o in tx.offsets((1, 2), 0)]
    d = _features(tx.Settings(weighting_norm="infinity")).to_dict()
    assert d["weighting_norm"] == "infinity" and not {"distances", "force2d_dimension", "offsets"} & set(d)
    keys = list(d)
    assert keys.index("weighting_norm") < keys.index("rows")


def test_json_writer_keeps_the_settings(tmp_path):
    from lungmask_b200.io import save_texture
    path = tmp_path / "t.json"
    save_texture(str(path), _features(tx.Settings((2,), 1)))
    d = json.loads(path.read_text())
    assert d["distances"] == [2] and d["force2d_dimension"] == 1 and len(d["offsets"]) == 8
    assert d["rows"][0]["gldm_counts"] == []


def _cli(tmp_path, argv):
    from lungmask_b200.__main__ import build_parser
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    return build_parser().parse_args([str(src), "out.nii", "--texture", str(tmp_path / "t.json")] + argv)


@pytest.mark.parametrize("argv,msg", [
    (["--texture-distances", "1,4"], "--texture-distances"), (["--texture-distances", "a"], "--texture-distances"),
    (["--texture-distances", ","], "--texture-distances")])
def test_cli_refusals(tmp_path, argv, msg):
    from lungmask_b200.__main__ import texture_settings_arguments
    with pytest.raises(SystemExit) as e:
        texture_settings_arguments(_cli(tmp_path, argv))
    assert msg in str(e.value)


@pytest.mark.parametrize("argv", [["--texture-force2d", "3"], ["--texture-weighting-norm", "chebyshev"]])
def test_cli_parser_refusals(tmp_path, argv):
    with pytest.raises(SystemExit):
        _cli(tmp_path, argv)


def test_cli_settings(tmp_path):
    from lungmask_b200.__main__ import texture_settings_arguments
    kw = texture_settings_arguments(_cli(tmp_path, []))
    assert tx.check_settings(**kw) == tx.Settings()
    kw = texture_settings_arguments(_cli(tmp_path, ["--texture-distances", "3,1", "--texture-force2d", "0",
                                                    "--texture-weighting-norm", "manhattan"]))
    assert tx.check_settings(**kw) == tx.Settings((1, 3), 0, "manhattan")


def test_cli_checks_before_segmentation(tmp_path, monkeypatch):
    import lungmask_b200.__main__ as cli

    def no_load(*a, **k):
        raise AssertionError("the input was read before the arguments were checked")
    monkeypatch.setattr(cli, "load_input_image", no_load)
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    for flag in ("--texture", "--wavelet", "--filtered"):
        with pytest.raises(SystemExit, match="--texture-distances"):
            cli.main([str(src), str(tmp_path / "out.nii"), flag, str(tmp_path / "t.json"), "--texture-distances", "5"])
