"""Mesh shape features per lung and lobe: the result of LMInferer.shape (lm_shape_sums_dev, lm_max_diameters_dev; DESIGN
§4.10).

Every row of `statistics` (each label l: mask == l, then "lung": mask != 0) is meshed by marching cubes on the mask padded
with one voxel of outside, as PyRadiomics does.  A cube is each 2x2x2 block of the padded grid; a vertex is the midpoint
of every cube edge whose two ends differ in membership.  The triangles of a cube follow from one face rule (see
triangle_table) and depend only on its 8-bit configuration, so the device counts, per row and configuration, the cubes
and the sum of their corner positions; SurfaceArea and MeshVolume follow exactly from those sums here.  The diameters are
the largest distances between mesh vertices; the principal axes come from exact integer moments of the voxel positions.
Everything here is pure numpy / Python in float64; the tests apply the same functions to reference sums.

Array axes (0, 1, 2) with spacing (s0, s1, s2) = spacing[::-1] (spacing is (x, y, z) in mm).  Corner k of a cube with
lowest corner p is p + ((k >> 2) & 1, (k >> 1) & 1, k & 1); configuration bit k is set when corner k is in the row.
"""
import functools
import math
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from .statistics import UNION

SHAPE_FEATURES = ("MeshVolume", "VoxelVolume", "SurfaceArea", "SurfaceVolumeRatio", "Sphericity", "Maximum3DDiameter",
                  "Maximum2DDiameterSlice", "Maximum2DDiameterColumn", "Maximum2DDiameterRow", "MajorAxisLength",
                  "MinorAxisLength", "LeastAxisLength", "Elongation", "Flatness")
DIAMETERS = ("Maximum3DDiameter", "Maximum2DDiameterSlice", "Maximum2DDiameterColumn", "Maximum2DDiameterRow")
# moments[r] of lm_shape_sums_dev: voxel count, then sums of the array indices (i, j, k) and their products
MOMENTS = ("N", "Si", "Sj", "Sk", "Sii", "Sjj", "Skk", "Sij", "Sik", "Sjk")
ROWS = 257   # row l = label l (row 0 stays zero), row 256 = mask != 0

CORNERS = np.array([((k >> 2) & 1, (k >> 1) & 1, k & 1) for k in range(8)], np.int64)
# edge e = (corner a, corner b, axis): axis 0 first, then 1, 2; within an axis by ascending a
EDGES = tuple((a, a | (4 >> m), m) for m in range(3) for a in range(8) if not a & (4 >> m))
# an edge midpoint in units of half a voxel, relative to the cube's lowest corner
EDGE_MID2 = np.array([CORNERS[a] + CORNERS[b] for a, b, _ in EDGES], np.int64)
_EDGE_OF = {(a, b): e for e, (a, b, _) in enumerate(EDGES)}


def _edge(a, b):
    return _EDGE_OF[(min(a, b), max(a, b))]


def _faces():
    """(outward normal in array axes, the face's 4 corners in cyclic order) for the 6 faces."""
    out = []
    for m in range(3):
        u, v = [x for x in range(3) if x != m]
        for s in (0, 1):
            cyc = []
            for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                c = np.zeros(3, np.int64)
                c[m], c[u], c[v] = s, du, dv
                cyc.append(int(c[0] * 4 + c[1] * 2 + c[2]))
            n = np.zeros(3, np.int64)
            n[m] = 2 * s - 1
            out.append((n, cyc))
    return out


FACES = _faces()


def face_segments(config):
    """The directed segments (edge, edge) of every cube face for `config`: one per face with two crossing edges, two
    (one cutting off each inside corner) when the face's inside corners are diagonal.  A segment a -> b is directed so
    that (b - a) x n points to the inside corner it separates, n the face's outward normal (array axes): the loops it
    forms then run so that their right-hand normal points out of the row in array axes.  The rule reads only the face's
    4 corners, so the two cubes of a face agree on its segments and traverse them in opposite directions."""
    inside = [(config >> k) & 1 for k in range(8)]
    segs = []
    for n, cyc in FACES:
        ins = [c for c in cyc if inside[c]]
        if len(ins) in (0, 4):
            continue
        if len(ins) == 2 and abs(cyc.index(ins[0]) - cyc.index(ins[1])) == 2:
            cuts = [(c, [_edge(c, cyc[(cyc.index(c) + 1) % 4]), _edge(c, cyc[(cyc.index(c) + 3) % 4])]) for c in ins]
        else:
            cross = [_edge(cyc[i], cyc[(i + 1) % 4]) for i in range(4) if inside[cyc[i]] != inside[cyc[(i + 1) % 4]]]
            cuts = [(ins[0], cross)]
        for c, (a, b) in cuts:
            d = EDGE_MID2[b] - EDGE_MID2[a]
            toward = 2 * CORNERS[c] - (EDGE_MID2[a] + EDGE_MID2[b]) / 2.0
            segs.append((a, b) if np.dot(np.cross(d, n), toward) > 0 else (b, a))
    return segs


def loops(config):
    """The closed loops of `config` as lists of edges, from chaining its face segments (each crossing edge lies on two
    faces, so it ends one segment and starts another).  Each loop starts at its lowest-numbered edge."""
    nxt = {}
    for a, b in face_segments(config):
        if a in nxt:
            raise AssertionError("config %d: edge %d starts two segments" % (config, a))
        nxt[a] = b
    out, seen = [], set()
    for s in sorted(nxt):
        if s in seen:
            continue
        lp, e = [], s
        while e not in seen:
            seen.add(e)
            lp.append(e)
            e = nxt[e]
        if e != s:
            raise AssertionError("config %d: the segments from edge %d do not close" % (config, s))
        out.append(lp)
    return out


_FACE_EDGES = [frozenset(_edge(cyc[i], cyc[(i + 1) % 4]) for i in range(4)) for _, cyc in FACES]


def _on_one_face(a, b):
    return any(a in f and b in f for f in _FACE_EDGES)


def fan_start(lp):
    """The fan vertex of a loop: its lowest-numbered edge whose fan diagonals join no two edges of one cube face (such
    a diagonal would lie in the face, where the neighbouring cube may draw the same one).  Every loop of the 256
    configurations has one."""
    for e in sorted(lp):
        s = lp.index(e)
        r = lp[s:] + lp[:s]
        if not any(_on_one_face(r[0], r[i]) for i in range(2, len(r) - 1)):
            return e
    raise AssertionError("loop %s: every fan has a diagonal in a face" % (lp,))


def _triangles(config):
    """Each loop as a fan from fan_start, reversed so that the right-hand normal points out of the row in (x, y, z) =
    (axis 2, axis 1, axis 0), a frame of the opposite handedness to the array axes."""
    tris = []
    for lp in loops(config):
        s = lp.index(fan_start(lp))
        lp = lp[s:] + lp[:s]
        tris += [(lp[0], lp[i + 1], lp[i]) for i in range(1, len(lp) - 1)]
    return tris


def triangle_table():
    """[256] lists of (edge, edge, edge) triangles, generated from the face rule (face_segments) and the fan rule
    (fan_start)."""
    return [_triangles(c) for c in range(256)]


TRIANGLES = triangle_table()


def config_geometry(spacing):
    """See _config_geometry (cached per spacing)."""
    return _config_geometry(tuple(float(s) for s in spacing))


@functools.lru_cache(maxsize=16)
def _config_geometry(spacing):
    """(area, n, w) per configuration for `spacing` (x, y, z) mm: area[c] = the summed triangle areas (mm^2), and with a',
    b', c' the triangle's vertices relative to the cube's lowest corner in (x, y, z) mm, n[c] = the sum over its
    triangles of a' x b' + b' x c' + c' x a' (mm^2, (x, y, z)) and w[c] = the sum of a' . (b' x c') (mm^3)."""
    sx, sy, sz = (float(s) for s in spacing)
    mid = EDGE_MID2[:, ::-1].astype(np.float64) * (0.5 * np.array([sx, sy, sz]))   # (x, y, z) mm
    area, nvec, w = np.zeros(256), np.zeros((256, 3)), np.zeros(256)
    for c, tris in enumerate(TRIANGLES):
        for ea, eb, ec in tris:
            a, b, d = mid[ea], mid[eb], mid[ec]
            area[c] += 0.5 * float(np.linalg.norm(np.cross(b - a, d - a)))
            nvec[c] += np.cross(a, b) + np.cross(b, d) + np.cross(d, a)
            w[c] += float(np.dot(a, np.cross(b, d)))
    return area, nvec, w


def mesh_area_volume(counts, possum, spacing, geometry=None):
    """(SurfaceArea mm^2, MeshVolume mm^3) of one row from its per-configuration cube counts [256] and corner-position
    sums [256][3] (array axes): A = sum_c count * area(c), V = (1/6) sum_c [n(c) . (S possum(c)) + count * w(c)], S the
    spacing as (x, y, z), each sum taken with math.fsum."""
    area, nvec, w = geometry if geometry is not None else config_geometry(spacing)
    sx, sy, sz = (float(s) for s in spacing)
    a_terms, v_terms = [], []
    for c in range(256):
        k = int(counts[c])
        if not k:
            continue
        px, py, pz = sx * float(possum[c][2]), sy * float(possum[c][1]), sz * float(possum[c][0])
        a_terms.append(k * area[c])
        v_terms += [nvec[c][0] * px, nvec[c][1] * py, nvec[c][2] * pz, k * w[c]]
    return math.fsum(a_terms), math.fsum(v_terms) / 6.0


def principal_moments(moments, spacing):
    """The eigenvalues (least, minor, major) of the population covariance (mm^2) of the voxel positions from the exact
    integer moments (MOMENTS order) and spacing (x, y, z).  N S_ab - S_a S_b is formed in Python integers and divided by
    N^2 with one rounding; eigenvalues in (-1e-10, 0) become 0 as in PyRadiomics."""
    m = [int(x) for x in moments]
    N = m[0]
    S = m[1:4]
    SS = {(0, 0): m[4], (1, 1): m[5], (2, 2): m[6], (0, 1): m[7], (0, 2): m[8], (1, 2): m[9]}
    s = [float(x) for x in spacing][::-1]
    C = np.zeros((3, 3))
    for (a, b), sab in SS.items():
        C[a, b] = C[b, a] = s[a] * s[b] * float(Fraction(N * sab - S[a] * S[b], N * N))
    ev = np.linalg.eigvalsh(C)
    ev = np.where((ev < 0) & (ev > -1e-10), 0.0, ev)
    return tuple(float(x) for x in ev)


def features(voxels, counts, possum, moments, d2, spacing, geometry=None):
    """The 14 SHAPE_FEATURES of one row from its exact sums and the four squared diameters d2 (3-D, slice, column, row);
    all NaN without voxels."""
    if voxels == 0:
        return {k: float("nan") for k in SHAPE_FEATURES}
    sx, sy, sz = (float(s) for s in spacing)
    A, V = mesh_area_volume(counts, possum, spacing, geometry)
    least, minor, major = principal_moments(moments, spacing)
    nan = float("nan")
    f = {"MeshVolume": V, "VoxelVolume": int(voxels) * sz * sy * sx, "SurfaceArea": A,
         "SurfaceVolumeRatio": A / V if V else nan, "Sphericity": (36.0 * math.pi * V * V) ** (1.0 / 3.0) / A if A else nan}
    for name, v in zip(DIAMETERS, d2):
        f[name] = math.sqrt(float(v))
    sq = lambda x: math.sqrt(x) if x >= 0 else nan
    f["MajorAxisLength"], f["MinorAxisLength"], f["LeastAxisLength"] = 4.0 * sq(major), 4.0 * sq(minor), 4.0 * sq(least)
    f["Elongation"] = sq(minor / major) if major > 0 else nan
    f["Flatness"] = sq(least / major) if major > 0 else nan
    return {k: float(f[k]) for k in SHAPE_FEATURES}


def check_spacing(spacing, what="shape"):
    """-> spacing (x, y, z) as 3 floats; ValueError when missing, of the wrong length, or not finite and positive."""
    if spacing is None:
        raise ValueError("%s: shape features need the voxel spacing; pass spacing=(x, y, z) in mm or a Volume / SimpleITK "
                         "image" % what)
    sp = tuple(float(s) for s in np.asarray(spacing, dtype=np.float64).reshape(-1))
    if len(sp) != 3 or not all(math.isfinite(s) and s > 0 for s in sp):
        raise ValueError("%s: spacing must be 3 finite positive sizes (x, y, z) in mm, got %s" % (what, spacing))
    return sp


# ---- numpy statements of what the device computes ---------------------------------------------------------------------
def _row_sel(mask, row):
    return mask != 0 if row == 256 else mask == row


def cube_sums_host(mask):
    """(cube_counts [257][256], cube_possum [257][256][3], moments [257][10]) int64 of a uint8 mask: the numpy statement
    of lm_shape_sums_dev."""
    mask = np.asarray(mask).view(np.uint8) if np.asarray(mask).dtype == bool else np.asarray(mask, np.uint8)
    n0, n1, n2 = mask.shape
    P = np.pad(mask, 1)
    corner = [P[d0:d0 + n0 + 1, d1:d1 + n1 + 1, d2:d2 + n2 + 1] for d0, d1, d2 in CORNERS]
    mixed = np.zeros(corner[0].shape, bool)
    for c in corner[1:]:
        mixed |= c != corner[0]
    idx = np.nonzero(mixed)
    C = np.stack([c[idx] for c in corner], axis=1)              # (m, 8) corner labels of the mixed cubes
    p = np.stack(idx, axis=1).astype(np.int64) - 1              # their lowest corners (array axes)
    counts = np.zeros((ROWS, 256), np.int64)
    possum = np.zeros((ROWS, 256, 3), np.int64)
    bits = (1 << np.arange(8)).astype(np.int64)

    def add(row, sel, conf):
        np.add.at(counts[row], conf, 1)
        for a in range(3):
            np.add.at(possum[row, :, a], conf, p[sel, a])

    for l in np.unique(C):
        if l == 0:
            continue
        eq = C == l
        sel = eq.any(axis=1)
        add(int(l), sel, (eq[sel] * bits).sum(axis=1))
    sel = (C == 0).any(axis=1)
    add(256, sel, ((C[sel] != 0) * bits).sum(axis=1))
    moments = np.zeros((ROWS, 10), np.int64)
    j = np.arange(n1, dtype=np.float64)[None, :]
    k = np.arange(n2, dtype=np.float64)
    for r in [int(x) for x in np.unique(mask) if x] + [256]:
        for z in range(0, n0, 16):   # per x-row: count, sum k, sum k^2 (float64 sums of integers below 2^53: exact)
            sel = _row_sel(mask[z:z + 16], r).astype(np.float64)
            i = np.arange(z, z + len(sel), dtype=np.float64)[:, None]
            cnt, sk, skk = sel.sum(axis=2), sel @ k, sel @ (k * k)
            v = [cnt.sum(), (i * cnt).sum(), (j * cnt).sum(), sk.sum(), (i * i * cnt).sum(), (j * j * cnt).sum(), skk.sum(),
                 (i * j * cnt).sum(), (i * sk).sum(), (j * sk).sum()]
            moments[r] += np.array(v).astype(np.int64)
    return counts, possum, moments


def mesh_vertices(member):
    """The doubled integer coordinates (m, 3) of every mesh vertex of a boolean (n0, n1, n2) row: u + v for each
    face-adjacent pair (u, v) of the padded grid that differ in membership."""
    M = np.pad(np.asarray(member, bool), 1)
    out = []
    for k in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[k], hi[k] = slice(0, -1), slice(1, None)
        idx = np.stack(np.nonzero(M[tuple(lo)] != M[tuple(hi)]), axis=1).astype(np.int64)
        c = 2 * idx - 2
        c[:, k] += 1
        out.append(c)
    return np.concatenate(out)


def _extreme_vertices(member):
    """(doubled coordinates (m, 3), 3-bit extremality) of the vertices that are the minimum or maximum on their line
    along some axis; bit j: along axis j."""
    M = np.pad(np.asarray(member, bool), 1)
    coords, masks = [], []
    for k in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[k], hi[k] = slice(0, -1), slice(1, None)
        E = M[tuple(lo)] != M[tuple(hi)]
        bits = np.zeros(E.shape, np.uint8)
        for j in range(3):
            n = E.shape[j]
            first = np.argmax(E, axis=j)
            last = n - 1 - np.argmax(np.flip(E, axis=j), axis=j)
            t = np.arange(n).reshape([-1 if a == j else 1 for a in range(3)])
            ext = (t == np.expand_dims(first, j)) | (t == np.expand_dims(last, j))
            bits |= (E & ext).astype(np.uint8) << j
        idx = np.nonzero(bits)
        c = 2 * np.stack(idx, axis=1).astype(np.int64) - 2
        c[:, k] += 1
        coords.append(c)
        masks.append(bits[idx])
    return np.concatenate(coords), np.concatenate(masks)


def pair_max_d2(X, spacing, block=2048):
    """The largest d^2 = ((D2 h2)^2 + (D1 h1)^2) + (D0 h0)^2 over all pairs of the doubled coordinates X (m, 3), h_k =
    s_k / 2 with (s0, s1, s2) = spacing[::-1]; every product and sum rounded on its own.  0.0 with fewer than 2 points."""
    X = np.asarray(X, np.int64)
    h = np.array([float(s) for s in spacing][::-1]) * 0.5
    best = 0.0
    for a in range(0, len(X), block):
        D = (X[a:a + block, None, :] - X[None, a:, :]).astype(np.float64)
        t0, t1, t2 = D[..., 0] * h[0], D[..., 1] * h[1], D[..., 2] * h[2]
        d2 = (t2 * t2 + t1 * t1) + t0 * t0
        if d2.size:
            best = max(best, float(d2.max()))
    return best


def _plane_max(X, axis, spacing, reduce=None):
    if not len(X):
        return 0.0
    order = np.argsort(X[:, axis], kind="stable")
    X = X[order]
    cuts = np.flatnonzero(np.diff(X[:, axis])) + 1
    return max(pair_max_d2(reduce(g, axis) if reduce else g, spacing) for g in np.split(X, cuts))


FAMILY_BITS = (7, 6, 5, 3)   # extremality bits each diameter family needs: all; axes 1, 2; axes 0, 2; axes 0, 1


def max_diameters_host(member, spacing, hull=False):
    """The squared diameters [3-D, slice, column, row] of a boolean row for `spacing` (x, y, z), over the vertices the device keeps (extreme
    on their lines along every axis of the family).  hull=True further reduces each set to the vertices of its
    scipy.spatial.ConvexHull (per plane for the 2-D families), which keeps the farthest pair."""
    X, bits = _extreme_vertices(member)
    red3 = red2 = None
    if hull:
        red3 = lambda P: _hull_vertices(P, None)
        red2 = lambda P, axis: _hull_vertices(P, axis)
    out = []
    for f, need in enumerate(FAMILY_BITS):
        P = X[(bits & need) == need]
        if f == 0:
            out.append(pair_max_d2(red3(P) if hull else P, spacing))
        else:
            out.append(_plane_max(P, f - 1, spacing, red2))
    return np.array(out)


def _hull_vertices(P, drop_axis):
    from scipy.spatial import ConvexHull
    Q = P if drop_axis is None else np.delete(P, drop_axis, axis=1)
    if len(Q) <= Q.shape[1] + 1:
        return P
    try:
        return P[ConvexHull(Q.astype(np.float64)).vertices]
    except Exception:   # a flat or collinear set: keep every point
        return P


def max_diameters_brute(member, spacing):
    """The squared diameters [3-D, slice, column, row] over every pair of mesh vertices (no pruning)."""
    V = mesh_vertices(member)
    return np.array([pair_max_d2(V, spacing)] + [_plane_max(V, a, spacing) for a in range(3)])


# ---- results ----------------------------------------------------------------------------------------------------------
def _json_value(v):
    return None if isinstance(v, float) and math.isnan(v) else v


@dataclass
class ShapeRow:
    label: object              # the label value (int), or "lung" for mask != 0
    name: str
    voxels: int
    features: dict = field(default_factory=dict)   # SHAPE_FEATURES -> float (NaN without voxels)
    cube_counts: np.ndarray = field(default_factory=lambda: np.zeros(256, np.int64))       # [256] cubes per configuration
    cube_possum: np.ndarray = field(default_factory=lambda: np.zeros((256, 3), np.int64))  # [256][3] sum of lowest corners
    moments: np.ndarray = field(default_factory=lambda: np.zeros(10, np.int64))           # MOMENTS
    d2: np.ndarray = field(default_factory=lambda: np.zeros(4, np.float64))               # squared DIAMETERS (mm^2)

    SUMMARY = ("label", "name", "voxels")

    def __getitem__(self, name):
        return self.features[name]

    def to_dict(self):
        d = {k: _json_value(getattr(self, k)) for k in self.SUMMARY}
        d["features"] = {k: _json_value(v) for k, v in self.features.items()}
        nz = np.flatnonzero(self.cube_counts)
        d["cube_counts"] = {str(int(c)): int(self.cube_counts[c]) for c in nz}
        d["cube_possum"] = {str(int(c)): [int(x) for x in self.cube_possum[c]] for c in nz}
        d["moments"] = dict(zip(MOMENTS, (int(x) for x in self.moments)))
        d["d2"] = dict(zip(DIAMETERS, (float(x) for x in self.d2)))
        return d


@dataclass
class ShapeFeatures:
    spacing: tuple             # (x, y, z) mm
    rows: list

    def __getitem__(self, label):
        """The row of a label value, or of "lung"."""
        for r in self.rows:
            if r.label == label:
                return r
        raise KeyError(label)

    def to_dict(self):
        """JSON-ready: NaN becomes None."""
        return {"spacing": list(self.spacing), "rows": [r.to_dict() for r in self.rows]}


def build_row(label, name, spacing, counts, possum, moments, d2, geometry=None):
    """The ShapeRow of row `label` (1..255, or 256 for "lung") from its exact sums and squared diameters."""
    voxels = int(moments[0])
    return ShapeRow(UNION if label == 256 else label, name, voxels,
                    features(voxels, counts, possum, moments, d2, spacing, geometry),
                    np.asarray(counts, np.int64).copy(), np.asarray(possum, np.int64).copy(),
                    np.asarray(moments, np.int64).copy(), np.asarray(d2, np.float64).copy())
