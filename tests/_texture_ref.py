"""Numpy reference matrices of the GLRLM, GLDM and NGTDM (lm_glrlm_dev, lm_neighbour_counts_dev) of a uint8 level map
(0 = outside the ROI): GLRLM by a run-position recurrence along each direction over shifted planes, GLDM / NGTDM by the
26 shifted slices of the zero-padded map.  The CPU tests check them against a voxel-by-voxel loop; the GPU tests and
tools/texture_cost.py compare the device matrices with them."""
import numpy as np

from lungmask_b200 import texture as tx

NB = tx.NEIGHBOURS


def glrlm_ref(L, ng):
    """int64 (13, ng, max(L.shape)): runs of level i + 1 and length k + 1 along each of tx.OFFSETS."""
    L = np.asarray(L)
    out = np.zeros((len(tx.OFFSETS), ng, max(L.shape)), np.int64)
    for d, off in enumerate(tx.OFFSETS):
        a = next(k for k in range(3) if off[k])            # the first non-zero component is +1
        rest = [k for k in range(3) if k != a]
        T = np.transpose(L, [a] + rest).astype(np.int32)
        e1, e2 = off[rest[0]], off[rest[1]]
        n0, n1, n2 = T.shape
        P = np.pad(T, ((1, 1), (1, 1), (1, 1)))
        R = np.zeros_like(P)                                 # position of the voxel within its run, 1-based
        for t in range(1, n0 + 1):
            cur = P[t, 1:n1 + 1, 1:n2 + 1]
            prev = P[t - 1, 1 - e1:n1 + 1 - e1, 1 - e2:n2 + 1 - e2]
            prev_r = R[t - 1, 1 - e1:n1 + 1 - e1, 1 - e2:n2 + 1 - e2]
            R[t, 1:n1 + 1, 1:n2 + 1] = np.where(cur > 0, np.where(prev == cur, prev_r + 1, 1), 0)
        cur = P[1:n0 + 1, 1:n1 + 1, 1:n2 + 1]
        succ = P[2:n0 + 2, 1 + e1:n1 + 1 + e1, 1 + e2:n2 + 1 + e2]
        end = (cur > 0) & (succ != cur)
        lev, length = cur[end], R[1:n0 + 1, 1:n1 + 1, 1:n2 + 1][end]
        out[d] = np.bincount((lev - 1) * out.shape[2] + length - 1, minlength=ng * out.shape[2]).reshape(ng, -1)
    return out


def neighbour_ref(L, ng, alpha):
    """(G, N, A), each int64 (ng, 27): dependence counts, NGTDM voxel counts and sums |W i - S| per (level, c or W)."""
    L = np.asarray(L).astype(np.int32)   # |W i - S| <= 26 * 255
    n0, n1, n2 = L.shape
    P = np.pad(L, 1)
    W, S, C = (np.zeros(L.shape, np.int32) for _ in range(3))
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                if dz == dy == dx == 0:
                    continue
                nb = P[1 + dz:n0 + 1 + dz, 1 + dy:n1 + 1 + dy, 1 + dx:n2 + 1 + dx]
                inroi = nb > 0
                W += inroi
                S += nb
                C += inroi & (np.abs(nb - L) <= alpha)
    roi = L > 0
    i = L[roi] - 1
    G = np.bincount(i * NB + C[roi], minlength=ng * NB).reshape(ng, NB)
    N = np.bincount(i * NB + W[roi], minlength=ng * NB).reshape(ng, NB)
    dev = np.abs(W[roi] * L[roi] - S[roi]).astype(np.float64)   # integers; every partial sum stays below 2^53
    A = np.bincount(i * NB + W[roi], weights=dev, minlength=ng * NB).astype(np.int64).reshape(ng, NB)
    return G, N, A
