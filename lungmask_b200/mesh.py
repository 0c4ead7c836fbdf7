"""Surface meshes per lung and lobe: the result of LMInferer.mesh (lm_mesh_counts_dev, lm_mesh_emit_dev; DESIGN §4.14).

The mesh of a row (label l: mask == l, or "lung": mask != 0) is the one LMInferer.shape measures (DESIGN §4.10): marching
cubes on the mask padded with one voxel of outside, one vertex at the midpoint of every cube edge whose ends differ in
membership, and the triangles of shape.triangle_table(), which is closed and outward-oriented.  Nothing is smoothed or
decimated.  Vertices are numbered by their edge: by grid point q in the padded grid's linear order (axis 0 slowest), then
edge axis m; triangles by cube in the same order, then table order.  Vertex positions are exact in half-voxel units
(index2 = 2q + e_m) and are placed in patient space as p = ((o + D[:, 0] (s_x x)) + D[:, 1] (s_y y)) + D[:, 2] (s_z z)
with (x, y, z) = index2[:, ::-1] / 2, every product and sum rounded on its own; "ras" negates the first two components.
When det D < 0 every triangle's last two vertices are swapped, so the normals still point out of the row.

mesh_host is the numpy statement of what the device computes; the tests compare the two bit for bit.
"""
import math
from dataclasses import dataclass

import numpy as np

from .shape import CORNERS, EDGES, TRIANGLES, check_spacing
from .statistics import UNION

SPACES = ("lps", "ras")
MAX_ELEMENTS = 2 ** 31 - 1   # int32 indices
IDENTITY = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)


def _table():
    """The triangle table as the C ABI takes it: offsets int32 [257] (configuration c owns triangles [off[c], off[c + 1]))
    and, per triangle vertex, the uint8 code (corner a << 2) | axis m of its cube edge."""
    off = np.zeros(257, np.int32)
    codes = []
    for c, tris in enumerate(TRIANGLES):
        off[c + 1] = off[c] + len(tris)
        for tri in tris:
            codes += [(EDGES[e][0] << 2) | EDGES[e][2] for e in tri]
    return off, np.array(codes, np.uint8)


TABLE_OFFSETS, TABLE_CODES = _table()


# ---- arguments --------------------------------------------------------------------------------------------------------
def check_space(space):
    if space not in SPACES:
        raise ValueError("mesh: space must be one of %s, got %r" % (", ".join(SPACES), space))
    return space


def _det(D):
    """det D in the order lm_mesh_emit_dev forms it (only its sign is used)."""
    return (D[0][0] * (D[1][1] * D[2][2] - D[1][2] * D[2][1]) - D[0][1] * (D[1][0] * D[2][2] - D[1][2] * D[2][0])
            + D[0][2] * (D[1][0] * D[2][1] - D[1][1] * D[2][0]))


def check_direction(direction):
    """-> the 3x3 direction (row-major, columns = image axes x, y, z) as nested float tuples; ValueError unless 9 finite
    values forming a matrix with |det| >= 1e-6."""
    d = np.asarray(IDENTITY if direction is None else direction, dtype=np.float64).reshape(-1)
    if d.size != 9 or not np.all(np.isfinite(d)):
        raise ValueError("mesh: direction must be 9 finite values (a row-major 3x3 matrix), got %s" % (direction,))
    D = tuple(tuple(float(x) for x in d[3 * r:3 * r + 3]) for r in range(3))
    if not abs(_det(D)) >= 1e-6:
        raise ValueError("mesh: the direction matrix %s is singular" % (D,))
    return D


def check_origin(origin):
    o = np.asarray((0.0, 0.0, 0.0) if origin is None else origin, dtype=np.float64).reshape(-1)
    if o.size != 3 or not np.all(np.isfinite(o)):
        raise ValueError("mesh: origin must be 3 finite values in mm, got %s" % (origin,))
    return tuple(float(x) for x in o)


def check_row(row):
    """-> the row number: a label 1..255, or 256 for "lung"."""
    if row == UNION:
        return 256
    if isinstance(row, (bool, np.bool_)) or not isinstance(row, (int, np.integer)) or not 1 <= int(row) <= 256:
        raise ValueError("mesh: a row is a label 1..255 or %r, got %r" % (UNION, row))
    return int(row)


def check_rows(rows):
    out = [check_row(r) for r in rows]
    if not out:
        raise ValueError("mesh: rows is empty")
    if len(set(out)) != len(out):
        raise ValueError("mesh: rows %s name a row twice" % (list(rows),))
    return out


def geometry(spacing=None, image=None):
    """(spacing (x, y, z), origin, direction 3x3) from `spacing` alone (origin 0, identity direction) or from a Volume /
    SimpleITK `image`, whose spacing `spacing` overrides."""
    origin, direction = None, None
    if image is not None:
        if spacing is None:
            spacing = tuple(image.spacing) if hasattr(image, "spacing") else tuple(image.GetSpacing())
        origin = tuple(image.origin) if hasattr(image, "origin") else tuple(image.GetOrigin())
        direction = tuple(image.GetDirection())
    return check_spacing(spacing, "mesh"), check_origin(origin), check_direction(direction)


def geometry_vector(spacing, origin, direction):
    """The 15 float64 of lm_mesh_emit_dev: origin, direction (row-major), spacing (x, y, z)."""
    return np.array(list(origin) + [x for r in direction for x in r] + list(spacing), np.float64)


def check_counts(label, n_vertices, n_triangles):
    if n_vertices > MAX_ELEMENTS or n_triangles > MAX_ELEMENTS:
        raise ValueError("mesh: row %r has %d vertices and %d triangles; int32 indices take at most 2^31 - 1"
                         % (label, n_vertices, n_triangles))


# ---- the numpy statement ----------------------------------------------------------------------------------------------
def place(index2, spacing, origin, direction, space="lps"):
    """float64 (V, 3) patient-space positions of the doubled coordinates index2 (V, 3)."""
    u = np.asarray(index2, np.int64).reshape(-1, 3)
    t = [float(spacing[k]) * (u[:, 2 - k].astype(np.float64) * 0.5) for k in range(3)]   # s_x x, s_y y, s_z z
    out = np.empty(u.shape, np.float64)
    for c in range(3):
        D = direction[c]
        out[:, c] = ((origin[c] + D[0] * t[0]) + D[1] * t[1]) + D[2] * t[2]
    if space == "ras":
        out[:, :2] = -out[:, :2]
    return out


def mesh_host(mask, row, spacing, origin=None, direction=None, space="lps", name=None):
    """The Mesh of `row` (a label 1..255, 256 or "lung") of a (n0, n1, n2) uint8 or bool mask: the numpy statement of
    lm_mesh_counts_dev + lm_mesh_emit_dev."""
    spacing, origin, direction = check_spacing(spacing, "mesh"), check_origin(origin), check_direction(direction)
    space, r = check_space(space), check_row(row)
    mask = np.asarray(mask)
    if mask.ndim != 3:
        raise ValueError("mesh: expected a (slices, H, W) mask, got shape %s" % (mask.shape,))
    M = np.pad(mask != 0 if r == 256 else mask == r, 1)   # padded grid point q at index q + 1
    keys = []
    for m in range(3):
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[m], hi[m] = slice(0, -1), slice(1, None)
        E = np.zeros(M.shape, bool)
        E[tuple(lo)] = M[tuple(lo)] != M[tuple(hi)]
        keys.append(np.flatnonzero(E).astype(np.int64) * 3 + m)
    keys = np.sort(np.concatenate(keys))                  # padded linear order of q, then m
    q = np.stack(np.unravel_index(keys // 3, M.shape), axis=1).astype(np.int64) - 1
    index2 = 2 * q + np.eye(3, dtype=np.int64)[keys % 3]
    # the cubes: lowest corner p at padded index p + 1, p_k in -1..n_k-1
    cube_shape = tuple(n - 1 for n in M.shape)
    conf = np.zeros(cube_shape, np.uint8)
    for k, (d0, d1, d2) in enumerate(CORNERS):
        conf |= M[d0:d0 + cube_shape[0], d1:d1 + cube_shape[1], d2:d2 + cube_shape[2]].astype(np.uint8) << k
    ntri = np.diff(TABLE_OFFSETS).astype(np.int64)
    conf = conf.reshape(-1)
    cubes = np.flatnonzero(ntri[conf])
    c = conf[cubes].astype(np.int64)
    k = ntri[c]
    first = np.cumsum(k) - k
    rows = np.repeat(TABLE_OFFSETS[c].astype(np.int64), k) + (np.arange(int(k.sum())) - np.repeat(first, k))
    codes = TABLE_CODES.reshape(-1, 3)[rows].astype(np.int64)
    pc = np.stack(np.unravel_index(np.repeat(cubes, k), cube_shape), axis=1).astype(np.int64)
    tris = np.empty(codes.shape, np.int64)
    for j in range(3):
        qa = pc + CORNERS[codes[:, j] >> 2]
        key = np.ravel_multi_index(tuple(qa.T), M.shape).astype(np.int64) * 3 + (codes[:, j] & 3)
        vid = np.searchsorted(keys, key)
        if len(key) and not np.array_equal(keys[np.minimum(vid, len(keys) - 1)], key):
            raise AssertionError("mesh: a triangle names an edge without a vertex")
        tris[:, j] = vid
    if _det(direction) < 0:
        tris[:, [1, 2]] = tris[:, [2, 1]]
    check_counts(UNION if r == 256 else r, len(keys), len(tris))
    return Mesh(UNION if r == 256 else r, name if name is not None else (UNION if r == 256 else "label %d" % r),
                place(index2, spacing, origin, direction, space), index2.astype(np.int32), tris.astype(np.int32), space)


# ---- results ----------------------------------------------------------------------------------------------------------
def _host(a):
    return a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)


@dataclass
class Mesh:
    label: object              # the label value (int), or "lung" for mask != 0
    name: str
    vertices: object           # float64 (V, 3) mm in `space`: numpy, or a CUDA tensor for a CUDA mask
    index2: object             # int32 (V, 3) doubled array-axis coordinates 2q + e_m
    triangles: object          # int32 (T, 3) vertex indices, outward by the right-hand rule
    space: str = "lps"

    @property
    def n_vertices(self):
        return int(self.vertices.shape[0])

    @property
    def n_triangles(self):
        return int(self.triangles.shape[0])

    def numpy(self):
        """The same mesh with numpy arrays."""
        return Mesh(self.label, self.name, _host(self.vertices), _host(self.index2), _host(self.triangles), self.space)

    def _corners(self):
        V, T = _host(self.vertices), _host(self.triangles).astype(np.int64)
        return V[T[:, 0]], V[T[:, 1]], V[T[:, 2]]

    def area(self):
        """The summed triangle areas (mm^2), math.fsum over the triangles."""
        a, b, c = self._corners()
        n = np.cross(b - a, c - a)
        return math.fsum(0.5 * np.sqrt(np.einsum("ij,ij->i", n, n)))

    def volume(self):
        """The enclosed volume (mm^3): math.fsum of a . (b x c) / 6 over the triangles, positions taken relative to the
        first vertex (a closed mesh's volume does not depend on that point)."""
        if not self.n_triangles:
            return 0.0
        a, b, c = self._corners()
        r = _host(self.vertices)[0]
        return math.fsum(np.einsum("ij,ij->i", a - r, np.cross(b - r, c - r))) / 6.0


@dataclass
class MeshSet:
    spacing: tuple             # (x, y, z) mm
    origin: tuple              # mm, in the frame of the image (LPS)
    direction: tuple           # 3x3, columns = image axes x, y, z
    space: str                 # "lps" or "ras": the frame of the vertices
    rows: list                 # Mesh per row

    def __getitem__(self, label):
        """The mesh of a label value, or of "lung"."""
        for r in self.rows:
            if r.label == label:
                return r
        raise KeyError(label)

    def __iter__(self):
        return iter(self.rows)

    def __len__(self):
        return len(self.rows)
