"""Voxel-based GLSZM, GLRLM, GLDM and NGTDM feature maps of one row: the result of LMInferer.texture_maps
(lm_texture_levels_dev, lm_texture_maps_dev; DESIGN §4.17), PyRadiomics' voxel-based extraction (voxelBased=True) of
those four classes.

The row, ROI, window W(c), candidates, centres, discretisation region D and level map are those of glcm_maps (DESIGN
§4.15, §4.16): a candidate is a voxel of W(c) with a non-zero level, a centre a candidate in the row; Np is the number of
candidates of W(c).  A neighbour, run step or zone link counts only when both voxels are candidates of W(c).
  GLSZM  the items are the zones: the 26-connected components of equal level among the candidates.
  GLRLM  per direction d of texture.OFFSETS, the items are the runs: maximal sequences of equal-level candidates along d.
  GLDM   the items are the candidates, each of size c + 1, c = its neighbours (of 26) that are candidates within
         gldm_alpha levels.
  NGTDM  for each candidate of level i with W >= 1 neighbours that are candidates, S their level sum: n_i += 1 and
         A(i, W) += |W i - S|.
An item has a level i and a size s (zone size, run length, dependence size); its key is i << 9 | s.

The zone-list evaluator of GLSZM, GLRLM (per direction) and GLDM (every product, sum and quotient rounded on its own;
cvt(k) the correctly rounded float64 of an integer; T = first_order_maps.entropy_table(K), K = (2r+1)^3, T[N][h] at
N (N - 1) / 2 + h - 1).  The items' keys are sorted; a run of c equal keys is the entry (i, s, c), entries ascending:
  integers   Nz = sum c, Si = sum c i, Si2 = sum c i^2, Ss = sum c s, Ss2 = sum c s^2, Sx = sum c i^2 s^2,
             Gi = sum_i (sum_s c)^2, Gs = sum_s (sum_i c)^2 (every sum exact)
  sums       over the entries ascending, each from 0.0: a1 + cvt(c) / cvt(s^2), a2 + cvt(c) / cvt(i^2),
             a3 + cvt(c) / cvt(i^2 s^2), a4 + cvt(c i^2) / cvt(s^2), a5 + cvt(c s^2) / cvt(i^2), ze + T[Nz][c]
  features   (texture.GLSZM_FEATURES order) SmallAreaEmphasis a1 / Nz, LargeAreaEmphasis cvt(Ss2) / Nz,
             GrayLevelNonUniformity cvt(Gi) / Nz, ...Normalized cvt(Gi) / cvt(Nz^2), SizeZoneNonUniformity cvt(Gs) / Nz,
             ...Normalized cvt(Gs) / cvt(Nz^2), ZonePercentage cvt(Nz) / cvt(Np),
             GrayLevelVariance cvt(Nz Si2 - Si^2) / cvt(Nz^2), ZoneVariance cvt(Nz Ss2 - Ss^2) / cvt(Nz^2),
             ZoneEntropy ze, LowGrayLevelZoneEmphasis a2 / Nz, HighGrayLevelZoneEmphasis cvt(Si2) / Nz,
             SmallAreaLowGrayLevelEmphasis a3 / Nz, SmallAreaHighGrayLevelEmphasis a4 / Nz,
             LargeAreaLowGrayLevelEmphasis a5 / Nz, LargeAreaHighGrayLevelEmphasis cvt(Sx) / Nz   (Nz as cvt(Nz))
GLSZM is the evaluator of the zones; GLDM the evaluator of the candidates, named by texture.GLDM_FEATURES (no
...Normalized gray level and no percentage); GLRLM the evaluator of each direction's runs, each feature summed over the
13 directions in direction order from 0.0 and divided by 13 (every centre has a run in every direction).
Bounds (r = 3, K = 343, i <= 255): sum c s = Np <= 343 for zones and runs, so Sx <= 255^2 343^2 ~ 7.7e9; dependence sizes
are at most 27, so Sx <= 255^2 27^2 343 ~ 1.6e10 and Nz Ss2 <= 343^2 27^2 ~ 8.6e7.  Every integer stays below 2^53, so
each cvt is exact.

NGTDM, with L = lcm(1..26) = 26771144400 (so L / W is an integer for W = 1..26), over the levels with n_i > 0 ascending:
  sigma_i = sum_W A(i, W) (L / W) <= 343 * 254 L ~ 2.3e15 < 2^52, so s_i = sigma_i / L; Nvp = sum n_i, Ngp the levels,
  X = sum n_i sigma_i <= 343 * 2.3e15 ~ 8e17, Sg = sum sigma_i, M1 = sum n_i i, M2 = sum n_i i^2, J1 = sum i, J2 = sum i^2,
  Q = 2 (Nvp M2 - M1^2) = sum_ij n_i n_j (i - j)^2, Y = 2 (Ngp M2 - 2 M1 J1 + Nvp J2) = sum_ij (n_i + n_j)(i - j)^2,
  B = 2 sum_{i<j} |i n_i - j n_j| (all int64)
  Coarseness  cvt(L Nvp) / cvt(X), 1e6 when X = 0
  Contrast    (cvt(Q) / cvt(Nvp^2 Ngp (Ngp - 1))) (cvt(Sg) / cvt(L Nvp)), 0 when Ngp = 1
  Busyness    cvt(X) / cvt(L B) (L B in 128 bits), 0 when B = 0
  Complexity  (sum over i < j ascending (i, then j) from 0.0 of cvt(2 (j - i)(n_i sigma_i + n_j sigma_j)) /
              cvt(L (n_i + n_j)), the numerator in 128 bits) / cvt(Nvp)
  Strength    cvt(L Y) / cvt(Nvp Sg) (L Y in 128 bits), 0 when Sg = 0
  all NaN when Nvp = 0.
maps_host is this sequence in numpy, vectorised over a chunk of ROI voxels; the device maps equal it bit for bit.
"""
import collections
import functools
from dataclasses import dataclass, field
from typing import ClassVar, Optional

import numpy as np

from . import texture as tx
from .first_order_maps import check_label, check_radius, entropy_table, region, roi_of
from .glcm_maps import level_map
from .statistics import UNION

CLASSES = ("glszm", "glrlm", "gldm", "ngtdm")
CLASS_FEATURES = {"glszm": tx.GLSZM_FEATURES, "glrlm": tx.GLRLM_FEATURES, "gldm": tx.GLDM_FEATURES,
                  "ngtdm": tx.NGTDM_FEATURES}
CLASS_CODES = {"glszm": 1, "glrlm": 2, "gldm": 3, "ngtdm": 4}   # LM_TEXMAP_* of lm_texture_maps_dev
LCM = 26771144400           # lcm(1..26)
_KEY_NONE = 1 << 20         # above every item key i << 9 | s
_GLDM_OF_GLSZM = tuple(tx.GLSZM_FEATURES.index(f) for f in tx._GLDM_AS_GLSZM)
_QUALIFIED = {"%s_%s" % (c, f): (c, k) for c in CLASSES for k, f in enumerate(CLASS_FEATURES[c])}


def check_classes(classes):
    """-> the classes in the order of CLASSES (texture.check_classes' rules); "glcm" is refused (glcm_maps has it)."""
    cls = tx.check_classes(classes)
    if "glcm" in cls:
        raise ValueError("classes: GLCM maps come from LMInferer.glcm_maps, not texture_maps")
    return cls


def check_features(features, classes):
    """-> the requested class-qualified names ("glszm_SmallAreaEmphasis") in class, then feature order: None for every
    feature of `classes` (checked), or a collection of names of those classes.  TypeError for a string, ValueError for an
    unknown name, a name of a class not requested, or an empty collection."""
    if features is None:
        return tuple("%s_%s" % (c, f) for c in classes for f in CLASS_FEATURES[c])
    if isinstance(features, (str, bytes)):
        raise TypeError("features must be a collection of names such as ('glszm_ZoneEntropy', 'ngtdm_Contrast'), got the "
                        "string %r" % (features,))
    want = list(features)
    for f in want:
        if f not in _QUALIFIED:
            raise ValueError("unknown feature %r; names are <class>_<Feature> such as glszm_SmallAreaEmphasis, with the "
                             "class one of %s" % (f, ", ".join(CLASSES)))
        if _QUALIFIED[f][0] not in classes:
            raise ValueError("feature %r is of class %s, which is not among the requested classes (%s)"
                             % (f, _QUALIFIED[f][0], ", ".join(classes)))
    if not want:
        raise ValueError("features is empty")
    return tuple("%s_%s" % (c, f) for c in classes for f in CLASS_FEATURES[c] if "%s_%s" % (c, f) in want)


def feature_bits(features, cls):
    """The feature bits of lm_texture_maps_dev for class `cls` of a checked feature tuple (bit k = the class's k-th
    feature); 0 when none of them is of that class."""
    return sum(1 << k for f, (c, k) in ((f, _QUALIFIED[f]) for f in features) if c == cls)


@dataclass
class TextureMaps:
    label: object              # the label value, or "lung"
    kernel_radius: int
    masked_kernel: bool
    bin_width: int
    init_value: float
    low: Optional[int]         # None without ROI voxels
    n_levels: int
    voxels: int                # ROI voxels
    classes: tuple
    gldm_alpha: int
    maps: dict = field(default_factory=collections.OrderedDict)   # "<class>_<Feature>" -> (S, H, W) float64
    FEATURE_CLASS: ClassVar[Optional[str]] = None   # the keys are already class-qualified (io.save_feature_maps)

    def __getitem__(self, feature):
        return self.maps[feature]

    def numpy(self):
        """A copy whose maps are numpy arrays."""
        m = collections.OrderedDict((k, v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in self.maps.items())
        return TextureMaps(self.label, self.kernel_radius, self.masked_kernel, self.bin_width, self.init_value, self.low,
                           self.n_levels, self.voxels, self.classes, self.gldm_alpha, m)


def maps_host(volume, mask, label=UNION, classes=CLASSES, features=None, kernel_radius=1, masked_kernel=True, bin_width=25,
              gldm_alpha=0, init_value=0.0, slices=None, chunk=2048):
    """The numpy statement of LMInferer.texture_maps (the module docstring's sequence) -> TextureMaps with numpy maps.
    `volume` (S, H, W) numeric, `mask` uint8 / bool.  `slices`: a range of output slices to compute (D still comes from
    the whole volume); the other slices hold init_value."""
    label = check_label(label)
    cls = check_classes(classes)
    feats = check_features(features, cls)
    r = check_radius(kernel_radius)
    bw = tx.check_arguments(bin_width)
    alpha = tx.check_alpha(gldm_alpha)
    vol = np.asarray(volume)
    if vol.dtype == np.float16:
        vol = vol.astype(np.float32)
    roi = roi_of(vol, mask, label)
    D = region(vol, roi, r, masked_kernel)
    lev, low, ng = level_map(vol, D, bw, "texture_maps: row %s" % label)
    n_roi = int(roi.sum())
    out = collections.OrderedDict((f, np.full(vol.shape, float(init_value), np.float64)) for f in feats)
    res = TextureMaps(label, r, bool(masked_kernel), bw, float(init_value), low if n_roi else None, ng if n_roi else 0,
                      n_roi, cls, alpha, out)
    if not n_roi:
        return res
    pad = np.pad(lev, r)
    zz, yy, xx = np.nonzero(roi)
    if slices is not None:
        keep = (zz >= slices.start) & (zz < slices.stop)
        zz, yy, xx = zz[keep], yy[keep], xx[keep]
    offs = [(dz, dy, dx) for dz in range(-r, r + 1) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]
    E = 2 * r + 1
    T = entropy_table(E ** 3)
    for c0 in range(0, len(zz), chunk):
        z, y, x = zz[c0:c0 + chunk] + r, yy[c0:c0 + chunk] + r, xx[c0:c0 + chunk] + r
        L = np.stack([pad[z + dz, y + dy, x + dx] for dz, dy, dx in offs], axis=1).astype(np.int64)
        for c in cls:
            f = window_features(c, L, E, T, alpha)
            for k, name in enumerate(CLASS_FEATURES[c]):
                q = "%s_%s" % (c, name)
                if q in out:
                    out[q][z - r, y - r, x - r] = f[k]
    return res


@functools.lru_cache(maxsize=None)
def _tables(E):
    """The window's geometry: (neighbours (K, 26) positions, K outside the window; per direction of texture.OFFSETS the
    step tables (E, K): position p + t d for t = 1..E-1, K outside; and the position p - d, K outside)."""
    K = E ** 3

    def at(z, y, x):
        return (z * E + y) * E + x if 0 <= z < E and 0 <= y < E and 0 <= x < E else K
    pos = [(z, y, x) for z in range(E) for y in range(E) for x in range(E)]
    nb = np.array([[at(z + a, y + b, x + c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1) if a or b or c]
                   for z, y, x in pos], np.int64)
    steps, prev = [], []
    for dz, dy, dx in tx.OFFSETS:
        steps.append(np.array([[at(z + t * dz, y + t * dy, x + t * dx) for z, y, x in pos] for t in range(1, E)],
                              np.int64).reshape(E - 1, K))
        prev.append(np.array([at(z - dz, y - dy, x - dx) for z, y, x in pos], np.int64))
    return nb, steps, prev


def _cvt(a):
    """cvt of an int64 or object (Python int) array: the correctly rounded float64."""
    return np.asarray(a).astype(np.float64)


def _seq_sum(t):
    """Sum of the columns of t (m, n) from 0.0 in column order (numpy's accumulate adds one column at a time)."""
    return np.add.accumulate(np.concatenate([np.zeros((t.shape[0], 1)), t], axis=1), axis=1)[:, -1]


def zone_features(keys, n_p, T):
    """The zone-list evaluator: keys (m, M) int64 item keys i << 9 | s (_KEY_NONE for no item), n_p (m,) Np ->
    (16, m) float64 in texture.GLSZM_FEATURES order.  Every window has an item."""
    m, M = keys.shape
    srt = np.sort(keys, axis=1)
    valid = srt < _KEY_NONE
    nz = valid.sum(axis=1).astype(np.int64)
    nxt = np.concatenate([srt[:, 1:], np.full((m, 1), -1)], axis=1)
    end = valid & (nxt != srt)
    pos = np.arange(M)[None, :]
    first = np.concatenate([np.ones((m, 1), bool), srt[:, 1:] != srt[:, :-1]], axis=1)
    start = np.maximum.accumulate(np.where(first, pos, 0), axis=1)
    c = np.where(end, pos + 1 - start, 0).astype(np.int64)
    i = np.where(end, srt >> 9, 1)
    s = np.where(end, srt & 511, 1)
    ii, ss = i * i, s * s
    Si, Si2, Ss, Ss2, Sx = ((c * w).sum(axis=1) for w in (i, ii, s, ss, ii * ss))
    rows = np.repeat(np.arange(m), M)
    gi = np.bincount(rows * 256 + (i & 255).ravel(), weights=c.ravel().astype(np.float64), minlength=m * 256)
    gs = np.bincount(rows * 512 + s.ravel(), weights=c.ravel().astype(np.float64), minlength=m * 512)
    Gi = (gi.astype(np.int64).reshape(m, 256) ** 2).sum(axis=1)   # counts <= 343: the float bincount is exact
    Gs = (gs.astype(np.int64).reshape(m, 512) ** 2).sum(axis=1)
    cf = _cvt(c)
    a1 = _seq_sum(np.where(end, cf / _cvt(ss), 0.0))
    a2 = _seq_sum(np.where(end, cf / _cvt(ii), 0.0))
    a3 = _seq_sum(np.where(end, cf / _cvt(ii * ss), 0.0))
    a4 = _seq_sum(np.where(end, _cvt(c * ii) / _cvt(ss), 0.0))
    a5 = _seq_sum(np.where(end, _cvt(c * ss) / _cvt(ii), 0.0))
    tb = nz * (nz - 1) // 2 - 1
    ze = _seq_sum(np.where(end, T[tb[:, None] + np.where(end, c, 1)], 0.0))
    N = _cvt(nz)
    NN = _cvt(nz * nz)
    return np.stack([a1 / N, _cvt(Ss2) / N, _cvt(Gi) / N, _cvt(Gi) / NN, _cvt(Gs) / N, _cvt(Gs) / NN, N / _cvt(n_p),
                     _cvt(nz * Si2 - Si * Si) / NN, _cvt(nz * Ss2 - Ss * Ss) / NN, ze, a2 / N, _cvt(Si2) / N, a3 / N,
                     a4 / N, a5 / N, _cvt(Sx) / N])


def _zone_keys(L, E, nb):
    """The GLSZM item keys of a chunk of windows: one per zone (26-connected, equal level), at the zone's first position."""
    m, K = L.shape
    Lx = np.concatenate([L, np.zeros((m, 1), np.int64)], axis=1)
    cand = L > 0
    link = cand[:, :, None] & (Lx[:, nb] == L[:, :, None])     # (m, K, 26): same level, both candidates
    big = np.int64(K)
    lab = np.where(cand, np.arange(K)[None, :], big)
    rows = np.arange(m)[:, None]
    while True:   # min-label propagation with pointer jumping: lab converges to the zone's first position
        labx = np.concatenate([lab, np.full((m, 1), big)], axis=1)
        new = np.minimum(lab, np.where(link, labx[:, nb], big).min(axis=2))
        new = np.where(cand, new[rows, np.minimum(new, K - 1)], big)
        if np.array_equal(new, lab):
            break
        lab = new
    size = np.bincount((rows * (K + 1) + lab).ravel(), minlength=m * (K + 1)).reshape(m, K + 1)[:, :K]
    root = cand & (lab == np.arange(K)[None, :])
    return np.where(root, (L << 9) | size, _KEY_NONE)


def _ngtdm(L, nb):
    """The five NGTDM features (5, m) of a chunk of windows (the module docstring's sequence)."""
    m, K = L.shape
    Lx = np.concatenate([L, np.zeros((m, 1), np.int64)], axis=1)
    Ln = Lx[:, nb]
    W = (Ln > 0).sum(axis=2)
    S = Ln.sum(axis=2)
    use = (L > 0) & (W > 0)
    a = np.abs(W * L - S) * (LCM // np.maximum(W, 1))   # <= 254 L per voxel
    key = (np.arange(m)[:, None] * 256 + L).ravel()
    n = np.bincount(key, weights=use.ravel().astype(np.float64), minlength=m * 256).reshape(m, 256).astype(np.int64)
    # every partial sum is an integer below 343 * 254 L < 2^53, so the float bincount is exact
    sig = np.bincount(key, weights=np.where(use, a, 0).ravel().astype(np.float64),
                      minlength=m * 256).reshape(m, 256).astype(np.int64)
    n[:, 0] = 0
    rows, cols = np.nonzero(n)
    per = np.bincount(rows, minlength=m)
    G = max(int(per.max()), 1)
    slot = np.arange(len(rows)) - np.repeat(np.cumsum(per) - per, per)
    lv = np.zeros((m, G), np.int64)
    nn = np.zeros((m, G), np.int64)
    sg = np.zeros((m, G), np.int64)
    lv[rows, slot], nn[rows, slot], sg[rows, slot] = cols, n[rows, cols], sig[rows, cols]
    ok = nn > 0
    nvp = nn.sum(axis=1)
    ngp = ok.sum(axis=1).astype(np.int64)
    X = (nn * sg).sum(axis=1)
    Sg = sg.sum(axis=1)
    M1, M2 = (nn * lv).sum(axis=1), (nn * lv * lv).sum(axis=1)
    J1, J2 = lv.sum(axis=1), (lv * lv).sum(axis=1)
    Q = 2 * (nvp * M2 - M1 * M1)
    Y = 2 * (ngp * M2 - 2 * M1 * J1 + nvp * J2)
    iN, nsg = lv * nn, nn * sg
    B = np.zeros(m, np.int64)
    comp = np.zeros(m)
    Lo = np.int64(LCM)
    for q in range(G - 1):
        j = slice(q + 1, G)
        pair = ok[:, q:q + 1] & ok[:, j]
        B = B + np.where(pair, np.abs(iN[:, q:q + 1] - iN[:, j]), 0).sum(axis=1)
        num = (2 * (lv[:, j] - lv[:, q:q + 1])).astype(object) * (nsg[:, q:q + 1] + nsg[:, j]).astype(object)
        den = Lo * np.where(pair, nn[:, q:q + 1] + nn[:, j], 1)
        comp = _seq_sum(np.concatenate([comp[:, None], np.where(pair, _cvt(num) / _cvt(den), 0.0)], axis=1))
    B = 2 * B
    some = nvp > 0
    nv1 = np.where(some, nvp, 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        coarse = np.where(X == 0, 1e6, _cvt(Lo * nv1) / _cvt(X))
        den_c = np.where(ngp > 1, nv1 * nv1 * ngp * (ngp - 1), 1)
        contrast = np.where(ngp > 1, (_cvt(Q) / _cvt(den_c)) * (_cvt(Sg) / _cvt(Lo * nv1)), 0.0)
        busy = np.where(B == 0, 0.0, _cvt(X) / _cvt(LCM * B.astype(object)))
        complexity = comp / _cvt(nv1)
        strength = np.where(Sg == 0, 0.0, _cvt(LCM * Y.astype(object)) / _cvt(nv1 * Sg))
    f = np.stack([coarse, contrast, busy, complexity, strength])
    return np.where(some[None, :], f, np.nan)


def window_features(cls, L, E, T, alpha=0):
    """The features (len(CLASS_FEATURES[cls]), m) of class `cls` of a chunk of windows: L (m, E^3) int64 levels in window
    order, 0 for a voxel that is not a candidate (or outside the array); T = entropy_table(E^3)."""
    nb, steps, prev = _tables(E)
    m, K = L.shape
    n_p = (L > 0).sum(axis=1)
    if cls == "glszm":
        return zone_features(_zone_keys(L, E, nb), n_p, T)
    if cls == "gldm":
        Lx = np.concatenate([L, np.zeros((m, 1), np.int64)], axis=1)
        Ln = Lx[:, nb]
        c = ((Ln > 0) & (np.abs(Ln - L[:, :, None]) <= alpha)).sum(axis=2)
        f = zone_features(np.where(L > 0, (L << 9) | (c + 1), _KEY_NONE), n_p, T)
        return f[list(_GLDM_OF_GLSZM)]
    if cls == "glrlm":
        Lx = np.concatenate([L, np.zeros((m, 1), np.int64)], axis=1)
        acc = np.zeros((len(tx.GLRLM_FEATURES), m))
        for st, pv in zip(steps, prev):
            start = (L > 0) & (Lx[:, pv] != L)
            run = np.ones((m, K), np.int64)
            cont = np.ones((m, K), bool)
            for t in range(E - 1):
                cont &= Lx[:, st[t]] == L
                run += cont
            acc = acc + zone_features(np.where(start, (L << 9) | run, _KEY_NONE), n_p, T)
        return acc / 13.0
    if cls == "ngtdm":
        return _ngtdm(L, nb)
    raise ValueError("unknown class %r" % (cls,))
