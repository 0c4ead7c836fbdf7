"""GLRLM, GLDM and NGTDM on the host: the known answer of a 5-voxel line, a voxel-by-voxel loop restatement of the three
matrices and of all 35 features (from PyRadiomics' definitions, the NGTDM's s_i as the sum of |i - mean neighbour
level|) against the numpy references of _texture_ref and the feature functions of lungmask_b200.texture, the matrix
identities, the argument checks and the writers (the default output keeps its keys and columns)."""
import csv
import itertools
import json
import math

import numpy as np
import pytest

from _texture_ref import glrlm_ref, neighbour_ref
from lungmask_b200 import io as lio
from lungmask_b200 import texture as tx

EPS = np.spacing(1)


# ---- loop restatement ------------------------------------------------------------------------------------------------
def _inside(shape, p):
    return all(0 <= p[k] < shape[k] for k in range(3))


def loop_runs(L):
    """[13 dicts {(level, length): runs}] from the definition: a run starts where the predecessor is not the same level."""
    out = []
    for off in tx.OFFSETS:
        runs = {}
        for v in itertools.product(*(range(n) for n in L.shape)):
            a = int(L[v])
            pred = tuple(v[k] - off[k] for k in range(3))
            if a == 0 or (_inside(L.shape, pred) and L[pred] == a):
                continue
            k, u = 1, tuple(v[q] + off[q] for q in range(3))
            while _inside(L.shape, u) and L[u] == a:
                k, u = k + 1, tuple(u[q] + off[q] for q in range(3))
            runs[(a, k)] = runs.get((a, k), 0) + 1
        out.append(runs)
    return out


def loop_neighbours(L, alpha):
    """{v: (level, W, S, c)} for every ROI voxel."""
    out = {}
    for v in itertools.product(*(range(n) for n in L.shape)):
        a = int(L[v])
        if a == 0:
            continue
        w = s = c = 0
        for d in itertools.product((-1, 0, 1), repeat=3):
            u = tuple(v[k] + d[k] for k in range(3))
            if d == (0, 0, 0) or not _inside(L.shape, u) or L[u] == 0:
                continue
            b = int(L[u])
            w, s, c = w + 1, s + b, c + (abs(b - a) <= alpha)
        out[v] = (a, w, s, c)
    return out


def loop_matrices(L, ng, alpha):
    runs = loop_runs(L)
    P = np.zeros((13, ng, max(L.shape)), np.int64)
    for d, r in enumerate(runs):
        for (a, k), n in r.items():
            P[d, a - 1, k - 1] = n
    G, N, A = (np.zeros((ng, 27), np.int64) for _ in range(3))
    for a, w, s, c in loop_neighbours(L, alpha).values():
        G[a - 1, c] += 1
        N[a - 1, w] += 1
        A[a - 1, w] += abs(w * a - s)
    return P, G, N, A


def loop_emphases(triples):
    """The 16 GLSZM-form values of {(i, j): count}, keyed by GLRLM name (GLDM maps onto them below)."""
    nr = sum(triples.values())
    np_ = sum(j * c for (i, j), c in triples.items())
    pg, pj = {}, {}
    for (i, j), c in triples.items():
        pg[i] = pg.get(i, 0) + c
        pj[j] = pj.get(j, 0) + c
    mi = sum(i * c / nr for (i, j), c in triples.items())
    mj = sum(j * c / nr for (i, j), c in triples.items())
    f = lambda g: sum(c * g(i, j) for (i, j), c in triples.items()) / nr   # noqa: E731
    return {
        "ShortRunEmphasis": f(lambda i, j: 1 / j ** 2), "LongRunEmphasis": f(lambda i, j: j ** 2),
        "GrayLevelNonUniformity": sum(x * x for x in pg.values()) / nr,
        "GrayLevelNonUniformityNormalized": sum(x * x for x in pg.values()) / nr ** 2,
        "RunLengthNonUniformity": sum(x * x for x in pj.values()) / nr,
        "RunLengthNonUniformityNormalized": sum(x * x for x in pj.values()) / nr ** 2,
        "RunPercentage": nr / np_,
        "GrayLevelVariance": f(lambda i, j: (i - mi) ** 2), "RunVariance": f(lambda i, j: (j - mj) ** 2),
        "RunEntropy": -sum(c / nr * math.log2(c / nr + EPS) for c in triples.values()),
        "LowGrayLevelRunEmphasis": f(lambda i, j: 1 / i ** 2), "HighGrayLevelRunEmphasis": f(lambda i, j: i ** 2),
        "ShortRunLowGrayLevelEmphasis": f(lambda i, j: 1 / (i ** 2 * j ** 2)),
        "ShortRunHighGrayLevelEmphasis": f(lambda i, j: i ** 2 / j ** 2),
        "LongRunLowGrayLevelEmphasis": f(lambda i, j: j ** 2 / i ** 2),
        "LongRunHighGrayLevelEmphasis": f(lambda i, j: i ** 2 * j ** 2),
    }


GLDM_FROM_RUN = dict(zip(tx.GLDM_FEATURES, (
    "ShortRunEmphasis", "LongRunEmphasis", "GrayLevelNonUniformity", "RunLengthNonUniformity",
    "RunLengthNonUniformityNormalized", "GrayLevelVariance", "RunVariance", "RunEntropy", "LowGrayLevelRunEmphasis",
    "HighGrayLevelRunEmphasis", "ShortRunLowGrayLevelEmphasis", "ShortRunHighGrayLevelEmphasis",
    "LongRunLowGrayLevelEmphasis", "LongRunHighGrayLevelEmphasis")))


def loop_features(L, alpha):
    """(glrlm, gldm, ngtdm) feature dicts from the loops alone."""
    runs = loop_runs(L)
    per = [loop_emphases(r) for r in runs]
    glrlm = {k: sum(p[k] for p in per) / len(per) for k in tx.GLRLM_FEATURES}
    nb = loop_neighbours(L, alpha)
    dep = {}
    for a, w, s, c in nb.values():
        dep[(a, c + 1)] = dep.get((a, c + 1), 0) + 1
    e = loop_emphases(dep)
    gldm = {k: e[r] for k, r in GLDM_FROM_RUN.items()}
    n, s_i = {}, {}
    for a, w, s, c in nb.values():
        if w:
            n[a] = n.get(a, 0) + 1
            s_i[a] = s_i.get(a, 0.0) + abs(a - s / w)
    nvp = sum(n.values())
    if nvp == 0:
        return glrlm, gldm, {k: float("nan") for k in tx.NGTDM_FEATURES}
    p = {i: n[i] / nvp for i in n}
    lv = sorted(p)
    ngp = len(lv)
    sum_ps = sum(p[i] * s_i[i] for i in lv)
    sum_s = sum(s_i.values())
    pairs = [(i, j) for i in lv for j in lv]
    busy = sum(abs(i * p[i] - j * p[j]) for i, j in pairs)
    ngtdm = {
        "Coarseness": 1e6 if sum_ps == 0 else 1 / sum_ps,
        "Contrast": 0.0 if ngp == 1 else
        sum(p[i] * p[j] * (i - j) ** 2 for i, j in pairs) / (ngp * (ngp - 1)) * sum_s / nvp,
        "Busyness": 0.0 if busy == 0 else sum_ps / busy,
        "Complexity": sum(abs(i - j) * (p[i] * s_i[i] + p[j] * s_i[j]) / (p[i] + p[j]) for i, j in pairs) / nvp,
        "Strength": 0.0 if sum_s == 0 else sum((p[i] + p[j]) * (i - j) ** 2 for i, j in pairs) / sum_s,
    }
    return glrlm, gldm, ngtdm


def close(a, b, tol=1e-12):
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def assert_features(got, want):
    assert list(got) == list(want) or set(got) == set(want)
    for k in want:
        assert close(got[k], want[k]), (k, got[k], want[k])


# ---- known answer ----------------------------------------------------------------------------------------------------
def test_known_answer_line():
    L = np.array([[[1, 1, 2, 2, 2]]], np.uint8)
    P = glrlm_ref(L, 2)
    assert P[0, 0, 1] == 1 and P[0, 1, 2] == 1 and P[0].sum() == 2
    for d in range(1, 13):
        assert P[d, 0, 0] == 2 and P[d, 1, 0] == 3 and P[d].sum() == 5
    f = tx.glrlm_features(P)
    assert f["ShortRunEmphasis"] == pytest.approx(0.936965811965812, rel=1e-15)
    assert f["LongRunEmphasis"] == pytest.approx(1.4230769230769231, rel=1e-15)
    assert f["RunPercentage"] == pytest.approx(0.9538461538461539, rel=1e-15)
    G, N, A = neighbour_ref(L, 2, 0)
    want = np.zeros((2, 27), np.int64)
    want[0, 1], want[1, 1], want[1, 2] = 2, 2, 1
    np.testing.assert_array_equal(G, want)
    g = tx.gldm_features(G)
    assert g["SmallDependenceEmphasis"] == pytest.approx(2 / 9, rel=1e-15)
    assert g["LargeDependenceEmphasis"] == pytest.approx(5.0, rel=1e-15)
    assert N[:, 0].sum() == 0 and list(N.sum(axis=1)) == [2, 3]
    s = [math.fsum(A[i, w] / w for w in range(1, 27)) for i in range(2)]
    assert s == [0.5, 0.5]
    n = tx.ngtdm_features(N, A)
    want_n = {"Coarseness": 2.0, "Contrast": 0.048, "Busyness": 0.3125, "Complexity": 0.2, "Strength": 2.0}
    for k, v in want_n.items():
        assert n[k] == pytest.approx(v, rel=1e-14), k
    assert list(n) == list(tx.NGTDM_FEATURES)
    assert len(tx.GLRLM_FEATURES) + len(tx.GLDM_FEATURES) + len(tx.NGTDM_FEATURES) == 35


# ---- random level maps -----------------------------------------------------------------------------------------------
def _maps():
    rng = np.random.default_rng(5)
    out = []
    for shape, ng, fill in (((3, 4, 5), 3, 0.8), ((4, 3, 6), 5, 0.5), ((2, 6, 4), 2, 1.0), ((5, 5, 3), 4, 0.3),
                            ((1, 7, 6), 6, 0.9), ((3, 1, 1), 2, 1.0)):
        L = rng.integers(1, ng + 1, shape).astype(np.uint8)
        L[rng.random(shape) >= fill] = 0
        out.append((L, ng))
    blob = np.zeros((4, 5, 6), np.uint8)          # a smooth ROI: long runs, many equal neighbours
    blob[1:4, 1:5, :5] = 2
    blob[2:, 2:, 2:] = 1
    blob[0, 0, 0] = 3                             # an isolated voxel
    out.append((blob, 3))
    return out


@pytest.mark.parametrize("alpha", [0, 1, 3])
@pytest.mark.parametrize("case", range(7))
def test_matrices_and_features_against_loops(case, alpha):
    L, ng = _maps()[case]
    P, G, N, A = loop_matrices(L, ng, alpha)
    np.testing.assert_array_equal(glrlm_ref(L, ng), P)
    for got, want in zip(neighbour_ref(L, ng, alpha), (G, N, A)):
        np.testing.assert_array_equal(got, want)
    glrlm, gldm, ngtdm = loop_features(L, alpha)
    if not L.any():
        return
    assert_features(tx.glrlm_features(P), glrlm)
    assert_features(tx.gldm_features(G), gldm)
    assert_features(tx.ngtdm_features(N, A), ngtdm)
    assert list(tx.glrlm_features(P)) == list(tx.GLRLM_FEATURES) and list(tx.gldm_features(G)) == list(tx.GLDM_FEATURES)


@pytest.mark.parametrize("case", range(7))
def test_matrix_identities(case):
    L, ng = _maps()[case]
    P = glrlm_ref(L, ng)
    n_p = int((L > 0).sum())
    k = np.arange(1, P.shape[2] + 1)
    assert int((P * k).sum()) == 13 * n_p
    for d in range(13):
        assert int((P[d] * k).sum(axis=1).sum()) == n_p
    hist = np.bincount(L.ravel(), minlength=ng + 1)[1:]
    G, N, A = neighbour_ref(L, ng, 1)
    np.testing.assert_array_equal(G.sum(axis=1), hist)
    np.testing.assert_array_equal(N.sum(axis=1), hist)
    isolated = sum(1 for a, w, s, c in loop_neighbours(L, 1).values() if w == 0)
    assert int(N[:, 0].sum()) == isolated and int(A[:, 0].sum()) == 0 and int(G[:, 0].sum()) >= isolated


def test_runs_from_counts_and_empty():
    L, ng = _maps()[1]
    P = glrlm_ref(L, ng)
    runs = tx.runs_from_counts(P)
    assert runs.shape[1] == 4 and (runs[:, 3] > 0).all()
    assert [tuple(r) for r in runs] == sorted(tuple(r) for r in runs)
    back = np.zeros_like(P)
    back[runs[:, 0], runs[:, 1] - 1, runs[:, 2] - 1] = runs[:, 3]
    np.testing.assert_array_equal(back, P)
    assert all(math.isnan(v) for v in tx.glrlm_features(np.zeros((13, 2, 3), np.int64)).values())
    assert all(math.isnan(v) for v in tx.gldm_features(np.zeros((2, 27), np.int64)).values())
    one = np.zeros((1, 27), np.int64)
    one[0, 0] = 1                                  # a single voxel: no neighbours, NGTDM NaN
    assert all(math.isnan(v) for v in tx.ngtdm_features(one, np.zeros_like(one)).values())
    assert tx.gldm_features(one)["SmallDependenceEmphasis"] == 1.0


def test_ngtdm_special_cases():
    N, A = np.zeros((3, 27), np.int64), np.zeros((3, 27), np.int64)
    N[1, 26] = 10                                  # a uniform ROI: one level, every s_i = 0
    f = tx.ngtdm_features(N, A)
    assert f == {"Coarseness": 1e6, "Contrast": 0.0, "Busyness": 0.0, "Complexity": 0.0, "Strength": 0.0}


# ---- rows, arguments, writers ------------------------------------------------------------------------------------------
def test_check_classes_and_alpha():
    assert tx.check_classes(["ngtdm", "glcm", "glrlm"]) == ("glcm", "glrlm", "ngtdm")
    assert tx.check_classes(("glszm", "glcm")) == tx.DEFAULT_CLASSES
    assert tx.check_classes(set(tx.CLASSES)) == tx.CLASSES
    with pytest.raises(ValueError, match="unknown"):
        tx.check_classes(["glcm", "firstorder"])
    with pytest.raises(ValueError, match="at least one"):
        tx.check_classes([])
    with pytest.raises(TypeError):
        tx.check_classes("glcm")
    with pytest.raises(TypeError):
        tx.check_classes([1])
    assert tx.check_alpha(0) == 0 and tx.check_alpha(np.int64(3)) == 3
    with pytest.raises(ValueError):
        tx.check_alpha(-1)
    for bad in (1.0, True, "1", None):
        with pytest.raises(TypeError):
            tx.check_alpha(bad)


def _features(classes, alpha=0):
    """A TextureFeatures of the loop maps as two rows plus an empty one, built from the numpy reference matrices."""
    rows = []
    for label, (L, ng) in ((1, _maps()[6]), (256, _maps()[1])):
        n = int((L > 0).sum())
        T = ng * (ng + 1) // 2
        rows.append(tx.build_row(label, "x", n, 25, -1000, ng, np.ones((13, T), np.int64), np.array([[1, n, 1]]), classes,
                                 glrlm_ref(L, ng), neighbour_ref(L, ng, alpha)))
    rows.insert(1, tx.build_row(2, "absent", 0, 25, classes=classes))
    return tx.TextureFeatures((1.0, 1.0, 2.0), 25, rows, tx.check_classes(classes), alpha)


OLD_ROW_KEYS = ["label", "name", "voxels", "low", "bin_width", "n_levels", "glcm", "glszm", "glszm_zones"]


def test_default_output_unchanged(tmp_path):
    d = _features(tx.DEFAULT_CLASSES).to_dict()
    assert list(d) == ["spacing", "bin_width", "rows"]
    assert all(list(r) == OLD_ROW_KEYS for r in d["rows"])
    res = _features(tx.DEFAULT_CLASSES)
    assert all(r.glrlm is None and r.gldm is None and r.ngtdm is None and r.glrlm_runs is None for r in res.rows)
    path = str(tmp_path / "t.csv")
    lio.save_texture(path, res)
    header = open(path).readline().strip().split(",")
    assert header == list(tx.TextureRow.SUMMARY) + ["glcm_" + k for k in tx.GLCM_FEATURES] + \
        ["glszm_" + k for k in tx.GLSZM_FEATURES]
    # the defaults of TextureFeatures and build_row are the default classes
    row = tx.build_row(1, "x", 0, 25)
    assert list(row.to_dict()) == OLD_ROW_KEYS
    assert list(tx.TextureFeatures(None, 25, [row]).to_dict()) == ["spacing", "bin_width", "rows"]


@pytest.mark.parametrize("classes", [tx.CLASSES, ("glrlm",), ("gldm", "glcm"), ("ngtdm",)])
def test_writers_new_classes(tmp_path, classes):
    res = _features(classes, alpha=2)
    d = res.to_dict()
    assert d["classes"] == list(tx.check_classes(classes))
    assert ("gldm_alpha" in d) == ("gldm" in classes) and d.get("gldm_alpha", 2) == 2
    for r, row in zip(d["rows"], res.rows):
        for c in tx.CLASSES:
            assert (c in r) == (c in classes), (c, classes)
        assert ("glrlm_runs" in r) == ("glrlm" in classes) and ("gldm_counts" in r) == ("gldm" in classes)
        assert ("ngtdm_sums" in r) == ("ngtdm" in classes) and ("glszm_zones" in r) == ("glszm" in classes)
        if "ngtdm" in classes and row.voxels:
            assert r["ngtdm_sums"] == row.ngtdm_sums.tolist() and np.asarray(r["ngtdm_counts"]).shape[1] == 27
    path = str(tmp_path / "t.json")
    lio.save_texture(path, res)
    assert json.load(open(path)) == json.loads(json.dumps(d))
    path = str(tmp_path / "t.csv")
    lio.save_texture(path, res)
    got = list(csv.DictReader(open(path)))
    names = {"glcm": tx.GLCM_FEATURES, "glszm": tx.GLSZM_FEATURES, "glrlm": tx.GLRLM_FEATURES, "gldm": tx.GLDM_FEATURES,
             "ngtdm": tx.NGTDM_FEATURES}
    want_cols = list(tx.TextureRow.SUMMARY) + ["%s_%s" % (c, k) for c in tx.check_classes(classes) for k in names[c]]
    assert list(got[0]) == want_cols
    for g, row in zip(got, res.rows):
        for c in tx.check_classes(classes):
            for k in names[c]:
                v = getattr(row, c)[k]
                assert (math.isnan(v) and g["%s_%s" % (c, k)] == "nan") or float(g["%s_%s" % (c, k)]) == v


def test_cli_rejects_bad_classes(tmp_path):
    from lungmask_b200.__main__ import main
    inp = tmp_path / "in.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    for bad in ("glcm,foo", ",", "GLCM"):
        with pytest.raises(SystemExit, match="--texture-classes"):
            main([str(inp), str(tmp_path / "m.npy"), "--texture", str(tmp_path / "t.csv"), "--texture-classes", bad])
