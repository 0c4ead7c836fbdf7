#!/usr/bin/env python
"""What the voxel-based GLCM maps cost: LMInferer.glcm_maps on CUDA tensors, the map kernel alone (lm_glcm_maps_dev)
and the write bound.

    python tools/glcm_maps_cost.py [--out DIR] [--rounds 3] [--radii 1,2,3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 phantoms of
oracle.synth (seed 100) at 300 slices of 256x256 and 512x512 with the two-lung mask of tools/statistics_cost.py, the
"lung" row and the lobe row 1, at each kernel radius of --radii, for all 22 features and for Contrast, JointEntropy, Idm:
  * "device"  LMInferer.glcm_maps on CUDA tensors, CUDA events on the current stream around the call (discretisation,
              level map and table upload included)
  * "kernel"  lm_glcm_maps_dev alone on the call's level map, CUDA events around it
  * "write_bound_ms"  features x 8 B x voxels at the H100 SXM data sheet's 3.35 TB/s, beside the kernel time
Median over alternating rounds and the spread (max - min).  The card name and power limit come from a read-only
nvidia-smi query.  Writes DIR/glcm_maps_cost.json when --out is given.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SLICES = 300
SUBSET = ("Contrast", "JointEntropy", "Idm")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for glcm_maps_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--radii", default="1,2,3", help="comma-separated kernel radii (default 1,2,3)")
    args = ap.parse_args()
    radii = [int(r) for r in args.radii.split(",")]

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, first_order_maps as fm, glcm_maps as gm, texture as tx
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="glcm_maps_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "int16 phantom (seed 100), 300-slice two-lung mask, bin width 25",
              "rounds": args.rounds, "unit": "ms", "cases": {}}

    def events(fn):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e)

    for hw in (256, 512):
        vol = synth.phantom(SLICES, hw, hw, seed=100)
        mask = lung_mask(SLICES, hw, hw)
        tv, tm = torch.from_numpy(vol).cuda(), torch.from_numpy(mask).cuda()
        for row in ("lung", 1):
            code = 256 if row == "lung" else row
            roi = mask > 0 if row == "lung" else mask == row
            n_roi = int(roi.sum())
            low, ng = tx.discretisation(float(vol[roi].min()), float(vol[roi].max()), 25)
            levels = torch.from_numpy(gm.level_map(vol, roi, 25)[0]).cuda()
            for r in radii:
                table = torch.from_numpy(fm.entropy_table(gm.max_pairs_n(r))).cuda()
                for feats in (None, SUBSET):
                    names = gm.check_features(feats)
                    out = torch.empty((len(names),) + vol.shape, dtype=torch.float64, device="cuda")

                    def kernel():
                        inferer.engine.glcm_maps_dev(levels.data_ptr(), tm.data_ptr(), vol.shape, code, r, ng, 0.0,
                                                     gm.feature_bits(names), table.data_ptr(), table.numel(),
                                                     out.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)

                    def device():
                        inferer.glcm_maps(tv, tm, label=row, features=feats, kernel_radius=r)

                    kernel()   # warm-up: module load
                    dev_t, ker_t = [], []
                    for _ in range(args.rounds):
                        ker_t.append(events(kernel))
                        dev_t.append(events(device))
                    del out
                    torch.cuda.empty_cache()
                    key = "%dx%d/%s/r%d/%s" % (hw, hw, row, r, "all" if feats is None else "subset")
                    c = {"roi_voxels": n_roi, "n_levels": ng, "maps": len(names),
                         "write_bound_ms": len(names) * 8 * vol.size / 3.35e12 * 1e3}
                    for name, ts in (("device", dev_t), ("kernel", ker_t)):
                        c[name] = {"median": float(np.median(ts)), "spread": float(np.ptp(ts))}
                    result["cases"][key] = c
                    print(key, json.dumps(c), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "glcm_maps_cost.json"), "w") as f:
            json.dump(result, f, indent=1)
    inferer.engine.close()


if __name__ == "__main__":
    main()
