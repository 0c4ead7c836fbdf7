#!/usr/bin/env python
"""What the regional statistics cost: LMInferer.regional_statistics on CUDA tensors and on numpy arrays, against scipy's
distance transform plus numpy statistics on the host.

    python tools/region_cost.py [--out DIR] [--rounds 3] [--host-rounds 1]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on 300-slice phantoms
(seed 100) at 256x256 and 512x512, each as int16 and as float32 (the int16 values plus a uniform fraction in [0, 1)),
with the two-lung mask of tools/statistics_cost.py, spacing (0.703125, 0.703125, 1.25) mm, the defaults: three zones by
volume, shells at 10 mm, Perc15 and LAA-950.  Per case:
  * "device"  regional_statistics on CUDA tensors (uploaded once), CUDA events on the current stream around the call
              (it ends with a synchronisation, so this is its whole span on the device timeline)
  * "edt"     surface_distance alone on the CUDA mask tensor, CUDA events
  * "numpy"   regional_statistics on the numpy arrays, wall time (the uploads included)
  * "host"    the same rows on the host: scipy.ndimage.distance_transform_edt, the zones of regions.zone_of_planes from
              np.bincount plane counts, then numpy mean / std / min / max / percentile / fraction below per row
              (--host-rounds rounds; the transform alone is reported as "host_edt")
Median over the rounds and the spread (max - min).  The device voxel counts of every row are checked against the host
ones.  The card name and power limit come from a read-only nvidia-smi query.  Writes DIR/region_cost.json with --out.
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


def host_rows(vol, mask):
    """{(row, region, index): (voxels, mean)} and the transform's seconds, computed on the host."""
    import scipy.ndimage as ndi
    from lungmask_b200 import regions as rg
    t0 = time.perf_counter()
    depth = np.float32(ndi.distance_transform_edt(mask > 0, sampling=SPACING[::-1]))
    t_edt = time.perf_counter() - t0
    v64 = vol.astype(np.float64)
    out = {}
    for row in (1, 2, "lung"):
        sel = mask > 0 if row == "lung" else mask == row
        counts = sel.reshape(sel.shape[0], -1).sum(axis=1)
        zone = rg.zone_of_planes(counts, 3, "volume", True)[:, None, None]
        parts = [("zone", k, sel & (zone == k)) for k in range(3)]
        parts += [("shell", 0, sel & (depth < np.float32(10.0))), ("shell", 1, sel & (depth >= np.float32(10.0)))]
        for region, k, part in parts:
            v = v64[part]
            out[(row, region, k)] = (int(v.size), v.mean(), v.std(), v.min(), v.max(), np.percentile(v, 15.0),
                                     (v < -950).mean())
    return out, t_edt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for region_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-rounds", type=int, default=1)
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="region_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    rng = np.random.default_rng(100)
    result = {"gpu": info, "workload": "300-slice phantoms seed 100, two-lung ellipsoid mask, spacing %s mm, 3 zones by "
              "volume, shells at 10 mm, Perc15, LAA-950" % (SPACING,), "rounds": args.rounds,
              "host_rounds": args.host_rounds, "unit": "ms", "cases": {}}
    print("\n%-24s %14s %14s %16s %16s %14s" % ("case", "device ms", "edt ms", "numpy-input ms", "host ms", "host edt ms"))
    for H in (256, 512):
        base = synth.phantom(SLICES, H, H, seed=100)
        mask = lung_mask(SLICES, H, H)
        for dt in ("int16", "float32"):
            vol = base if dt == "int16" else (base + rng.random(base.shape, dtype=np.float32)).astype(np.float32)
            name = "%dx%dx%d %s" % (SLICES, H, H, dt)
            tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
            torch.cuda.synchronize()
            inferer.regional_statistics(tv, tm, spacing=SPACING)     # warm-up: work buffers, module load
            inferer.regional_statistics(vol, mask, spacing=SPACING)
            dev, edt, npy, host, host_edt = [], [], [], [], []
            for _ in range(args.rounds):
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                r_dev = inferer.regional_statistics(tv, tm, spacing=SPACING)
                e1.record()
                inferer.surface_distance(tm, SPACING[::-1])
                e2.record()
                e2.synchronize()
                dev.append(e0.elapsed_time(e1))
                edt.append(e1.elapsed_time(e2))
                t0 = time.perf_counter()
                inferer.regional_statistics(vol, mask, spacing=SPACING)
                npy.append((time.perf_counter() - t0) * 1e3)
            for _ in range(args.host_rounds):
                t0 = time.perf_counter()
                want, t_edt = host_rows(vol, mask)
                host.append((time.perf_counter() - t0) * 1e3)
                host_edt.append(t_edt * 1e3)
            for (row, region, k), w in want.items():
                assert r_dev.row(row, region, k).stats.voxels == w[0], (name, row, region, k)
            series = {"device": dev, "edt": edt, "numpy": npy, "host": host, "host_edt": host_edt}
            med = {k: float(np.median(v)) for k, v in series.items()}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in series.items()}
            result["cases"][name] = {"median": med, "spread": spread, "rounds": series}
            print("%-24s %7.2f (%5.2f) %7.2f (%5.2f) %8.1f (%5.1f) %8.0f (%5.0f) %8.0f (%4.0f)" % (
                name, med["device"], spread["device"], med["edt"], spread["edt"], med["numpy"], spread["numpy"],
                med["host"], spread["host"], med["host_edt"], spread["host_edt"]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "region_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
