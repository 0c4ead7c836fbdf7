"""Numpy reference matrices of the generalised neighbourhoods (lm_glcm_offsets_dev, lm_neighbour_offsets_dev,
lm_zone_sizes_plane_dev; DESIGN §4.18) of a uint8 level map (0 = outside the ROI): GLCM by slicing and np.bincount per
offset, GLDM / NGTDM by the shifted slices of the map zero-padded by 3, in-plane zones by scipy.ndimage.label per level
with the 3x3 in-plane structure.  The CPU tests check them against voxel-by-voxel loops; the GPU tests and
tools/texture_settings_cost.py compare the device matrices with them."""
import numpy as np

PAD = 3


def glcm_offsets_ref(L, ng, offs):
    """int64 (len(offs), ng (ng + 1) / 2): U_o(i <= j) per offset, in np.triu_indices order."""
    L = np.asarray(L)
    T = ng * (ng + 1) // 2
    U = np.zeros((len(offs), T), np.int64)
    n = L.shape
    for d, off in enumerate(offs):
        if any(abs(o) >= n[k] for k, o in enumerate(off)):
            continue   # no pair fits along that axis
        src = tuple(slice(max(0, -o), n[k] - max(0, o)) for k, o in enumerate(off))
        dst = tuple(slice(max(0, o), n[k] - max(0, -o)) for k, o in enumerate(off))
        a, b = L[src].astype(np.int64), L[dst].astype(np.int64)
        both = (a > 0) & (b > 0)
        i, j = np.minimum(a, b)[both], np.maximum(a, b)[both]
        U[d] = np.bincount((i - 1) * ng - (i - 1) * (i - 2) // 2 + (j - i), minlength=T)
    return U


def neighbour_offsets_ref(L, ng, alpha, offs):
    """(G, N, A), each int64 (ng, 2 len(offs) + 1), over the neighbours v +- o."""
    L = np.asarray(L).astype(np.int32)
    cols = 2 * len(offs) + 1
    n0, n1, n2 = L.shape
    P = np.pad(L, PAD)
    W, S, C = (np.zeros(L.shape, np.int32) for _ in range(3))
    for off in offs:
        for sgn in (1, -1):
            dz, dy, dx = (sgn * o for o in off)
            nb = P[PAD + dz:n0 + PAD + dz, PAD + dy:n1 + PAD + dy, PAD + dx:n2 + PAD + dx]
            inroi = nb > 0
            W += inroi
            S += nb
            C += inroi & (np.abs(nb - L) <= alpha)
    roi = L > 0
    i = L[roi] - 1
    G = np.bincount(i * cols + C[roi], minlength=ng * cols).reshape(ng, cols)
    N = np.bincount(i * cols + W[roi], minlength=ng * cols).reshape(ng, cols)
    dev = np.abs(W[roi] * L[roi] - S[roi]).astype(np.float64)   # integers; every partial sum stays below 2^53
    A = np.bincount(i * cols + W[roi], weights=dev, minlength=ng * cols).astype(np.int64).reshape(ng, cols)
    return G, N, A


def plane_structure(axis):
    """The 3x3x3 structure of 8-connectivity within the planes normal to `axis`."""
    st = np.zeros((3, 3, 3), bool)
    idx = [slice(None)] * 3
    idx[axis] = 1
    st[tuple(idx)] = True
    return st


def zones_ref(L, structure):
    """(k, 3) int64 (level, size, count) triples of the zones of equal level under `structure`, sorted."""
    import scipy.ndimage as ndi
    L = np.asarray(L)
    zones = []
    for lv in range(1, int(L.max()) + 1 if L.size else 1):
        lab, k = ndi.label(L == lv, structure)
        if k:
            s, c = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
            zones += [(lv, int(x), int(y)) for x, y in zip(s, c)]
    return np.array(zones, np.int64).reshape(-1, 3)
