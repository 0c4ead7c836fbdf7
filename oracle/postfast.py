"""A fast, exact restatement of `restate.postprocessing` (utils.py:272-358).  TEST INFRASTRUCTURE ONLY.

`restate.postprocessing` relabels the whole volume for every merge candidate (`regionmask[regionmask == r] = t`), so
its cost is O(candidates x voxels) and it stops being usable at a few thousand speckles.  This module computes the same
result - bit for bit, taps included - in about O(N log N + sum of ring sizes), so that the CUDA post-processing can be
compared with it at benchmark sizes (hundreds of thousands of regions, 78 M voxels):

  * regions are labelled once (`standins.cc_label`); the 6-neighbour pairs that cross a region boundary are listed
    once, grouped by the region they leave: (neighbour voxel, the neighbour's original region id)
  * a merge only redirects ids: `cur[orig] -> current id`, and the current id keeps the list of its original members
  * a candidate's ring is the union of its members' boundary pairs, each neighbour voxel counted once, minus the
    voxels that belong to the candidate itself.  That is the reference's one-voxel 6-connected dilation inside the
    margin-2 box: the margin always covers the dilation, so the box changes nothing.
  * everything else - the stable area order, records, the `to_label` table, the cached-area and record growth of the
    target, the target rule (ascending ids, strict `>`, so the lowest id wins ties; ids equal to a spare label VALUE are
    skipped, as the reference does) and step 6 - is the reference's arithmetic unchanged.

`diag` (optional dict) receives what the CUDA merge loop's schedule would see on this input (postproc.cu,
merge_loop_mc_kernel): the region count, the candidates, the largest number of distinct non-zero neighbour ids of any
candidate, and the batch lengths of the default multi-CTA schedule.  tests/test_postfast_host.py checks the schedule
against tests/test_merge_batches.py's emulation and the result against `restate.postprocessing`.
"""
import numpy as np
from scipy import ndimage

from . import restate
from .standins import cc_label

# the merge loop's gates (lungmask_b200/csrc/postproc.cu)
MC_SMALL = 192      # up to this many regions one CTA runs the plain sequential loop
MC_WINDOW = 2048    # order positions classified per build step
MC_BMAX = 256       # members per batch
MC_HASH = 1024      # distinct neighbour ids a batch member's table holds; above that the serial routine decides it
SORT_SMEM = 4096    # region_sort_kernel sorts in shared memory up to this many regions

_SMALL_RING = 512   # rings up to this many pairs are counted in plain Python, larger ones with numpy


def boundary_pairs(reg: np.ndarray):
    """For every foreground voxel q and 6-neighbour p with reg[p] != reg[q]: the pair (reg[q], p), grouped by reg[q].
    -> (offsets, neighbour voxel, neighbour's region id): region r's pairs are [offsets[r], offsets[r + 1])."""
    S, H, W = reg.shape
    flat = reg.ravel()
    src, nbv = [], []
    for ax, step in ((0, H * W), (1, W), (2, 1)):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[ax], hi[ax] = slice(None, -1), slice(1, None)
        a, b = reg[tuple(lo)], reg[tuple(hi)]
        diff = a != b
        for side, other in ((a, step), (b, -step)):   # q on the low side (neighbour + step), then on the high side
            zz, yy, xx = np.nonzero(diff & (side > 0))
            q = (zz * H + yy) * W + xx
            if other < 0:
                q = q + step     # the high side sits one step further along the axis
            src.append(flat[q])
            nbv.append(q + other)
        del diff
    src = np.concatenate(src) if src else np.zeros(0, np.int64)
    nbv = np.concatenate(nbv) if nbv else np.zeros(0, np.int64)
    order = np.argsort(src, kind="stable")
    src, nbv = src[order], nbv[order]
    R = int(flat.max()) if flat.size else 0
    offsets = np.zeros(R + 2, np.int64)
    np.cumsum(np.bincount(src, minlength=R + 1), out=offsets[1:])
    return offsets, nbv, flat[nbv]


def postprocessing(label_image: np.ndarray, spare=(), skip_below: int = 3, taps: dict = None, diag: dict = None) -> np.ndarray:
    """restate.postprocessing, with the same arguments and taps; `diag` as in the module docstring."""
    spare = list(spare)
    spare_set = {int(s) for s in spare}
    lab = np.asarray(label_image)
    reg = cc_label(lab)
    if taps is not None:
        taps["regions0"] = reg.copy()
    flat = reg.ravel()
    R = int(flat.max()) if flat.size else 0
    if diag is not None:
        diag.update(regions=R, candidates=0, max_ids=0, batches=[], serial=0,
                    schedule="sequential" if R <= MC_SMALL else "batched", sort="smem" if R <= SORT_SMEM else "global")
    origlabels = np.unique(lab)
    record = [0] * (int(origlabels.max()) + 1)
    to_label = np.zeros(R + 1, np.uint8)
    cur = list(range(R + 1))
    if R:
        area = np.bincount(flat, minlength=R + 1).tolist()
        val = np.zeros(R + 1, np.int64)
        val[flat] = lab.ravel()
        value = val.tolist()
        order = (np.argsort(np.asarray(area[1:]), kind="stable") + 1).tolist()   # regions.sort(key=area), stable
        for r in order:
            v = value[r]
            if area[r] > record[v]:
                record[v] = area[r]
                to_label[r] = v
        offsets, nbv, nbo = boundary_pairs(reg)
        offsets = offsets.tolist()
        members = {}
        sched = _Schedule(reg, order, area, value, record, spare_set, skip_below) if diag is not None and R > MC_SMALL else None
        for p, r in enumerate(order):
            if sched is not None:
                sched.reach(p)
            v = value[r]
            a = area[r]
            if not ((a < record[v] or v in spare_set) and a >= skip_below):
                continue
            mem = members.get(r, (r,))
            cnt = _ring_counts(r, mem, offsets, nbv, nbo, cur)
            target, best = r, 0
            for n in sorted(cnt):
                c = cnt[n]
                if n != 0 and c > best and n not in spare_set:
                    best, target = c, n
            if diag is not None:
                ids = len(cnt) - (0 in cnt)
                diag["candidates"] += 1
                diag["max_ids"] = max(diag["max_ids"], ids)
                if sched is not None:
                    sched.member(p, ids)
            if target == r:
                continue
            for m in mem:
                cur[m] = target
            tm = members.get(target)
            if tm is None:
                tm = members[target] = [target]
            tm.extend(mem)
            members.pop(r, None)
            before = area[target]
            tv = value[target]
            if before == record[tv]:
                record[tv] += a
            area[target] = before + a
            if sched is not None:
                sched.merged(p, r, target, before)
        if sched is not None:
            diag["batches"], diag["serial"] = sched.batches, sched.serial
    cur = np.asarray(cur, np.int64)
    lut = to_label[cur]
    lut[np.isin(lut, spare)] = 0
    mapped = lut[reg]
    if taps is not None:
        taps["regions1"] = cur[reg]
        taps["mapped"] = mapped.copy()
    return restate.finish_labels(mapped)


def _ring_counts(r, mem, offsets, nbv, nbo, cur):
    """{current id: ring voxels} of the region r made of the original regions `mem` (0 = background)."""
    n = sum(offsets[m + 1] - offsets[m] for m in mem)
    if n <= _SMALL_RING:
        ring = {}
        for m in mem:
            s, e = offsets[m], offsets[m + 1]
            if e > s:
                ring.update(zip(nbv[s:e].tolist(), nbo[s:e].tolist()))
        cnt = {}
        for o in ring.values():
            c = cur[o]
            if c != r:
                cnt[c] = cnt.get(c, 0) + 1
        return cnt
    if len(mem) == 1:
        vox, org = nbv[offsets[r]:offsets[r + 1]], nbo[offsets[r]:offsets[r + 1]]
    else:
        vox = np.concatenate([nbv[offsets[m]:offsets[m + 1]] for m in mem])
        org = np.concatenate([nbo[offsets[m]:offsets[m + 1]] for m in mem])
    _, first = np.unique(vox, return_index=True)
    u, inv = np.unique(org[first], return_inverse=True)
    ids = np.asarray([cur[x] for x in u.tolist()], np.int64)[inv]
    ids, counts = np.unique(ids[ids != r], return_counts=True)
    return dict(zip(ids.tolist(), counts.tolist()))


class _Schedule:
    """The batch schedule of merge_loop_mc_kernel followed alongside the sequential loop.  Batches give the sequential
    loop's result (tests/test_merge_batches.py), so the tables at a batch's first position are the sequential loop's
    tables there; the build step reads them, the members' merges are then applied in order.

    build: from position k, classify the order (windows of MC_WINDOW positions until one holds a candidate); list the
    candidates from the first one up to the first non-candidate with area >= skip_below (a record growth could turn it
    into a candidate) or the window's end; keep at most MC_BMAX, and cut before the first member whose box is not a
    voxel apart from an earlier member's.  apply: a merge that lifts a region of the batch's span over skip_below ends
    the batch there; a member with more than MC_HASH neighbour ids ends it at its own position, which the serial routine
    processes alone."""

    def __init__(self, reg, order, area, value, record, spare_set, skip):
        self.order, self.area, self.value, self.record = order, area, value, record
        self.spare, self.skip = spare_set, skip
        self.pos = {r: i for i, r in enumerate(order)}
        self.box = {}
        for i, sl in enumerate(ndimage.find_objects(reg), start=1):
            self.box[i] = [sl[0].start, sl[0].stop, sl[1].start, sl[1].stop, sl[2].start, sl[2].stop]
        self.batches, self.serial = [], 0
        self.next, self.end = 0, 0     # where the next batch is built; the end of the current batch's span

    def _cls(self, q):
        r = self.order[q]
        a, v = self.area[r], self.value[r]
        if a < self.skip:
            return 0
        return 1 if (a < self.record[v] or v in self.spare) else 2

    def reach(self, p):
        if p < self.next:
            return
        R = len(self.order)
        ws, first, boxes, q = p, None, [], p
        while q < R:
            if q >= ws + MC_WINDOW:
                if first is not None:
                    break
                ws = q
            c = self._cls(q)
            if c == 2 and first is not None:
                break
            if c == 1:
                if len(boxes) == MC_BMAX:
                    break
                b = np.asarray(self.box[self.order[q]])
                if boxes:
                    B = np.asarray(boxes)
                    sep = ((B[:, 0::2] >= b[1::2] + 1) | (b[0::2] >= B[:, 1::2] + 1)).any(1)
                    if not sep.all():
                        break
                if first is None:
                    first = q
                boxes.append(b.tolist())
            q += 1
        self.end = self.next = q
        if boxes:
            self.batches.append(len(boxes))

    def member(self, p, ids):
        if ids > MC_HASH and p < self.next:
            self.serial += 1
            self.next = min(self.next, p + 1)

    def merged(self, p, r, t, before):
        b, c = self.box[t], self.box[r]
        self.box[t] = [min(b[0], c[0]), max(b[1], c[1]), min(b[2], c[2]), max(b[3], c[3]), min(b[4], c[4]), max(b[5], c[5])]
        pt = self.pos[t]
        if before < self.skip <= self.area[t] and p < pt < self.end and pt < self.next:
            self.next = pt
