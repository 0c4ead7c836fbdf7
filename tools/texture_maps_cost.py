#!/usr/bin/env python
"""What the voxel-based GLSZM, GLRLM, GLDM and NGTDM maps cost: LMInferer.texture_maps on CUDA tensors, the map kernel
alone (lm_texture_maps_dev) and the write bound.

    python tools/texture_maps_cost.py [--out DIR] [--rounds 3] [--radii 1,2,3] [--sizes 256,512]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 phantoms of
oracle.synth (seed 100) at 300 slices of each size of --sizes with the two-lung mask of tools/statistics_cost.py, the
"lung" row and the lobe row 1, each class alone with all its features, at each kernel radius of --radii:
  * "device"  LMInferer.texture_maps on CUDA tensors, CUDA events on the current stream around the call (discretisation,
              level map and table upload included)
  * "kernel"  lm_texture_maps_dev alone on the call's level map, CUDA events around it
  * "write_bound_ms"  features x 8 B x voxels at the H100 SXM data sheet's 3.35 TB/s, beside the kernel time
Median over alternating rounds and the spread (max - min); r = 3 runs one round.  The card name and power limit come
from a read-only nvidia-smi query in the same run.  Writes DIR/texture_maps_cost.json when --out is given.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for texture_maps_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--radii", default="1,2,3", help="comma-separated kernel radii (default 1,2,3)")
    ap.add_argument("--sizes", default="256,512", help="comma-separated slice sizes (default 256,512)")
    args = ap.parse_args()
    radii = [int(r) for r in args.radii.split(",")]

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, first_order_maps as fm, glcm_maps as gm, texture as tx, texture_maps as tmaps
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="texture_maps_cost_")
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

    for hw in (int(x) for x in args.sizes.split(",")):
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
                table = torch.from_numpy(fm.entropy_table((2 * r + 1) ** 3)).cuda()
                for cls in tmaps.CLASSES:
                    names = tmaps.check_features(None, (cls,))
                    out = torch.empty((len(names),) + vol.shape, dtype=torch.float64, device="cuda")

                    def kernel():
                        inferer.engine.texture_maps_dev(levels.data_ptr(), tm.data_ptr(), vol.shape, code, r, ng,
                                                        tmaps.CLASS_CODES[cls], 0, 0.0, tmaps.feature_bits(names, cls),
                                                        table.data_ptr(), table.numel(), out.data_ptr(),
                                                        stream=torch.cuda.current_stream().cuda_stream)

                    def device():
                        inferer.texture_maps(tv, tm, classes=(cls,), label=row, kernel_radius=r)

                    kernel()   # warm-up: module load
                    dev_t, ker_t = [], []
                    for _ in range(args.rounds if r < 3 else 1):
                        ker_t.append(events(kernel))
                        dev_t.append(events(device))
                    del out
                    torch.cuda.empty_cache()
                    key = "%dx%d/%s/r%d/%s" % (hw, hw, row, r, cls)
                    c = {"roi_voxels": n_roi, "n_levels": ng, "maps": len(names), "rounds": len(ker_t),
                         "write_bound_ms": len(names) * 8 * vol.size / 3.35e12 * 1e3}
                    for name, ts in (("device", dev_t), ("kernel", ker_t)):
                        c[name] = {"median": float(np.median(ts)), "spread": float(np.ptp(ts))}
                    result["cases"][key] = c
                    print(key, json.dumps(c), flush=True)
                    if args.out:   # written as it goes, so a cut-short run keeps what it measured
                        os.makedirs(args.out, exist_ok=True)
                        with open(os.path.join(args.out, "texture_maps_cost.json"), "w") as f:
                            json.dump(result, f, indent=1)
    inferer.engine.close()


if __name__ == "__main__":
    main()
