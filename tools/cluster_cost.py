#!/usr/bin/env python
"""What the LAA cluster size distributions cost: LMInferer.laa_clusters on CUDA tensors and on numpy arrays, against
scipy on the host.

    python tools/cluster_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on two 300-slice phantoms
(seed 100) at 256x256 and 512x512, each as int16 and as float32 (the int16 values plus a uniform fraction in [0, 1)),
with the two-lung mask of tools/statistics_cost.py, LAA-950 clusters at connectivity 6 and 26.  Two more int16 cases at
512x512 exercise the paths that many or large clusters take: "speckle" (3.5 % of the voxels set to -1000 HU: some 10^5
clusters of one voxel, the shared-memory small-size bins) and "bulla" (a ball of radius 60 at -1000 HU in the right
lung: one cluster of about 9 x 10^5 voxels, every one of its voxels' size atomics on one root).  Per case:
  * "device"  LMInferer.laa_clusters on CUDA tensors (uploaded once), CUDA events on the current stream around the call;
              the call ends with a synchronisation, so this is its whole span on the device timeline (the bincount of
              the mask that finds its labels included)
  * "engine"  the same, the lm_laa_clusters_dev call alone (Engine.laa_clusters_dev)
  * "numpy"   LMInferer.laa_clusters on the numpy arrays, wall time (the uploads and the mask's bincount included)
  * "scipy"   the same rows on the host: scipy.ndimage.label + np.bincount + np.unique for both lungs and the union
Median over the rounds and the spread (max - min).  Every device result is checked against the scipy one (all pairs).
The card name and power limit come from a read-only nvidia-smi query.  Writes DIR/cluster_cost.json when --out is given.
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
THRESHOLD = -950


def scipy_rows(vol, mask, conn):
    import scipy.ndimage as ndi
    st = np.ones((3, 3, 3), bool) if conn == 26 else ndi.generate_binary_structure(3, 1)
    laa = (mask > 0) & (vol < THRESHOLD)
    out = {}
    for row in (1, 2, "lung"):
        sel = laa if row == "lung" else laa & (mask == row)
        lab, _ = ndi.label(sel, st)
        out[row] = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for cluster_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="cluster_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    rng = np.random.default_rng(100)
    result = {"gpu": info, "workload": "300-slice phantoms seed 100, two-lung ellipsoid mask, LAA-950 clusters",
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    print("\n%-34s %14s %14s %16s %16s %10s %10s" % ("case", "device ms", "engine ms", "numpy-input ms", "scipy ms",
                                                     "clusters", "laa %"))
    cases = []
    for H in (256, 512):
        base = synth.phantom(SLICES, H, H, seed=100)
        mask = lung_mask(SLICES, H, H)
        for dt in ("int16", "float32"):
            vol = base if dt == "int16" else (base + rng.random(base.shape, dtype=np.float32)).astype(np.float32)
            cases.append(("%dx%dx%d %s" % (SLICES, H, H, dt), vol, mask))
    speckle = base.copy()
    speckle[rng.random(base.shape) < 0.035] = -1000
    cases.append(("%dx512x512 int16 speckle" % SLICES, speckle, mask))
    z, y, x = np.ogrid[:SLICES, :512, :512]
    bulla = base.copy()
    bulla[(z - SLICES // 2) ** 2 + (y - 256) ** 2 + (x - int(0.32 * 512)) ** 2 <= 60 * 60] = -1000
    cases.append(("%dx512x512 int16 bulla" % SLICES, bulla, mask))
    for case, vol, mask in cases:
        tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
        torch.cuda.synchronize()
        code = 0 if vol.dtype == np.int16 else 1
        for conn in (6, 26):
            name = "%s conn %d" % (case, conn)
            inferer.laa_clusters(tv, tm, connectivity=conn)     # warm-up: work buffers, module load
            inferer.laa_clusters(vol, mask, connectivity=conn)
            dev, eng, npy, host = [], [], [], []
            for _ in range(args.rounds):
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                r_dev = inferer.laa_clusters(tv, tm, connectivity=conn)
                e1.record()
                inferer.engine.laa_clusters_dev(tv.data_ptr(), code, tm.data_ptr(), vol.shape, THRESHOLD, conn,
                                                stream=torch.cuda.current_stream().cuda_stream)
                e2.record()
                e2.synchronize()
                dev.append(e0.elapsed_time(e1))
                eng.append(e1.elapsed_time(e2))
                launches = inferer.engine.last_timings()["kernel_launches"]
                t0 = time.perf_counter()
                r_np = inferer.laa_clusters(vol, mask, connectivity=conn)
                npy.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                want = scipy_rows(vol, mask, conn)
                host.append((time.perf_counter() - t0) * 1e3)
                for row, (s, c) in want.items():
                    for r in (r_dev, r_np):
                        assert np.array_equal(r[row].sizes, s) and np.array_equal(r[row].counts, c), (name, row)
            med = {k: float(np.median(v)) for k, v in (("device", dev), ("engine", eng), ("numpy", npy), ("scipy", host))}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in (("device", dev), ("engine", eng), ("numpy", npy),
                                                                     ("scipy", host))}
            lung = r_dev["lung"]
            result["cases"][name] = {"median": med, "spread": spread, "kernel_launches": launches,
                                     "clusters": lung.clusters, "laa_fraction": lung.laa_voxels / float((mask > 0).sum()),
                                     "pairs": int(lung.sizes.size), "d": lung.d,
                                     "rounds": {"device": dev, "engine": eng, "numpy": npy, "scipy": host}}
            print("%-34s %7.2f (%5.2f) %7.2f (%5.2f) %8.1f (%5.1f) %8.0f (%5.0f) %10d %10.2f" % (
                name, med["device"], spread["device"], med["engine"], spread["engine"], med["numpy"], spread["numpy"],
                med["scipy"], spread["scipy"], lung.clusters, 100 * lung.laa_voxels / float((mask > 0).sum())), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cluster_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
