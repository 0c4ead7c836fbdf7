#!/usr/bin/env python
"""What the mesh shape features cost: LMInferer.shape on CUDA tensors and on numpy arrays, the two C entry points alone,
the diameter candidates per row, and the same sums and diameters on the host with numpy / scipy.

    python tools/shape_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, at 300 slices of 256x256 and
512x512, on the two-lung mask of tools/statistics_cost.py (rows 1, 2 and "lung") and on a five-lobe split of it (rows
1..5 and "lung"), spacing (0.703125, 0.703125, 1.25) mm.  Per case:
  * "device"     LMInferer.shape on a CUDA tensor, CUDA events on the current stream around the call; it ends with a
                 synchronisation, so this is its whole span on the device timeline
  * "sums"       lm_shape_sums_dev alone (Engine.shape_sums_dev), CUDA events around the call
  * "diameters"  lm_max_diameters_dev alone for every row, CUDA events around each call (the sum, and the slowest row)
  * "numpy"      LMInferer.shape on the numpy mask, wall time (the upload included)
  * "host"       one round on the host: shape.cube_sums_host and, per row, shape.max_diameters_host with the convex-hull
                 reduction (a brute-force search over the candidates alone would be ~10^10 pairs per row)
  * candidates   per row, the vertices the 3-D and the slice family keep, of all mesh vertices (counted on the host)
Median over the rounds and the spread (max - min).  The device sums are checked against the host sums and the device
diameters against the host diameters.  The card name and power limit come from a read-only nvidia-smi query.  Writes
DIR/shape_cost.json when --out is given.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SLICES = 300
SPACING = (0.703125, 0.703125, 1.25)   # (x, y, z) mm


def lobes_of(mask):
    """Five lobes: label 1 split into 1 (upper half of the slices), 2 and 3 (front / back of the lower half), label 2
    into 4 (upper half) and 5."""
    S, H, _ = mask.shape
    z, y, _ = np.ogrid[:S, :H, :1]
    lobes = mask.copy()
    lobes[(mask == 1) & (z >= S // 2)] = 2
    lobes[(mask == 1) & (z >= S // 2) & (y >= H // 2)] = 3
    lobes[(mask == 2) & (z < S // 2)] = 4
    lobes[(mask == 2) & (z >= S // 2)] = 5
    return lobes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for shape_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, shape as sh

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="shape_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "300-slice two-lung ellipsoid mask and its five-lobe split, spacing %s" % (SPACING,),
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    s_arr = SPACING[::-1]
    print("\n%-20s %5s %14s %13s %16s %16s %9s  %s" % ("case", "rows", "device ms", "sums ms", "diameters ms (max)",
                                                      "numpy-input ms", "host ms", "candidates 3-D / slice / vertices"))
    for H in (256, 512):
        two = lung_mask(SLICES, H, H)
        for which, mask in (("lungs", two), ("lobes", lobes_of(two))):
            name = "%dx%dx%d %s" % (SLICES, H, H, which)
            rows = [int(x) for x in np.unique(mask) if x] + [256]
            tm = torch.from_numpy(mask).to("cuda:0")
            stream = torch.cuda.current_stream().cuda_stream
            inferer.shape(tm, spacing=SPACING)     # warm-up: work buffers, module load
            inferer.shape(mask, spacing=SPACING)
            t0 = time.perf_counter()
            want_sums = sh.cube_sums_host(mask)
            want_d2 = {r: sh.max_diameters_host((mask != 0) if r == 256 else (mask == r), SPACING, hull=True) for r in rows}
            host = (time.perf_counter() - t0) * 1e3
            cands = {}
            for r in rows:
                member = (mask != 0) if r == 256 else (mask == r)
                _, bits = sh._extreme_vertices(member)
                cands[str(r)] = [int(((bits & 7) == 7).sum()), int(((bits & 6) == 6).sum()), int(len(sh.mesh_vertices(member)))]
            dev, sums, diam, diam_max, npy = [], [], [], [], []
            for _ in range(args.rounds):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3 + len(rows))]
                ev[0].record()
                r_dev = inferer.shape(tm, spacing=SPACING)
                ev[1].record()
                got = inferer.engine.shape_sums_dev(tm.data_ptr(), mask.shape, stream=stream)
                ev[2].record()
                d2 = {}
                for k, r in enumerate(rows):
                    d2[r] = inferer.engine.max_diameters_dev(tm.data_ptr(), mask.shape, r, s_arr, stream=stream)
                    ev[3 + k].record()
                ev[-1].synchronize()
                dev.append(ev[0].elapsed_time(ev[1]))
                sums.append(ev[1].elapsed_time(ev[2]))
                per = [ev[2 + k].elapsed_time(ev[3 + k]) for k in range(len(rows))]
                diam.append(sum(per))
                diam_max.append(max(per))
                t0 = time.perf_counter()
                r_np = inferer.shape(mask, spacing=SPACING)
                npy.append((time.perf_counter() - t0) * 1e3)
                for a, b in zip(("cube_counts", "cube_possum", "moments"), want_sums):
                    assert np.array_equal(got[a], b), (name, a)
                for r in rows:
                    assert np.array_equal(d2[r], want_d2[r]), (name, r, d2[r], want_d2[r])
                assert json.dumps(r_dev.to_dict()) == json.dumps(r_np.to_dict()), name
            series = (("device", dev), ("sums", sums), ("diameters", diam), ("diameters_max_row", diam_max), ("numpy", npy))
            med = {k: float(np.median(v)) for k, v in series}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in series}
            med["host"] = host
            result["cases"][name] = {"median": med, "spread": spread, "rows": rows, "candidates": cands,
                                     "rounds": {k: v for k, v in series}}
            print("%-20s %5d %7.2f (%5.2f) %6.2f (%4.2f) %7.2f (%6.2f) %8.1f (%5.1f) %9.0f  %s" % (
                name, len(rows), med["device"], spread["device"], med["sums"], spread["sums"], med["diameters"],
                med["diameters_max_row"], med["numpy"], spread["numpy"], host,
                " ".join("%s:%d/%d/%d" % (r, *c) for r, c in cands.items())), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "shape_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
